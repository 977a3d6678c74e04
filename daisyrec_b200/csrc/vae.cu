// vae.cu -- Multi-VAE (daisy/model/VAECFRecommender.py) on the device: fp32 on CUDA cores, every sum in a fixed order and no
// floating-point atomics, so two fits from the same inputs are bitwise equal.
//
// Parameters live in one flat fp32 block in module order (encoder layers, then decoder layers; per layer W then b).  The first
// encoder layer's weight is stored item-major [I, H0] (the transpose of nn.Linear's [H0, I]), so its forward pass is a gather of
// the batch items' rows and its gradient touches only those rows.  The last decoder layer's weight is nn.Linear's [I, H] as is.
//
// One step (calc_loss :92-110 + backward + optimizer.step):
//   input     the batch users' rows of the input CSR (drb_vae_input_csr), L2-normalised, dropped (host bits or Philox),
//             and grouped by item for the first layer's weight gradient
//   encoder   layer 0 as a sparse gather in slot order, the others on gemm_nt
//   reparam   z = mu + eps * exp(logvar / 2) and the KL row sums, one kernel
//   decoder   gemm_nt; the output layer's logits are replaced in place by dz = (softmax(z) sum(r) - r) / B (vae_ce_kernel)
//   backward  weight gradients on gemm_tn (written, no split-K), input gradients on gemm_nn (the output layer's K = I one split
//             into fixed slices summed in order), bias gradients by ordered column sums, layer 0 per item in row order
//   update    dense_update over the whole block (torch.optim.Adam / SGD are dense: untouched rows still move)
#include "common.cuh"
#include "gemm.cuh"
#include "step.cuh"

namespace drb {

constexpr int kVaeMaxHidden = 8;
constexpr int kVaeMaxItems = 1 << 20;        // the per-row dedup bitmap of the input CSR (I bits) must fit shared memory
constexpr int kVaeInputThreads = 32;         // one warp per history row in the input CSR kernels
constexpr int kVaeMaxBatch = 32768;          // rows per step: vae_dw0_kernel holds a bitmap and an index per row in shared memory
constexpr size_t kVaeDw0MaxSmem = sizeof(uint32_t) * (kVaeMaxBatch / 32) + sizeof(int) * kVaeMaxBatch;

struct VaeDims {
    int I = 0, nh = 0, lat = 0, half = 0, ne = 0, nd = 0;
    int e[kVaeMaxHidden + 2], d[kVaeMaxHidden + 2];          // encoder / decoder widths
    long long w_off[2 * kVaeMaxHidden + 2], b_off[2 * kVaeMaxHidden + 2];   // layer L: encoder L < ne, decoder ne + l
    long long nW = 0;
    int maxw = 0;                                           // widest activation other than the logits
    int slices = 1;                                         // k slices of the output layer's input gradient (K = I)
};

static bool vae_dims(VaeDims &v, int I, const int32_t *hidden, int nh, int lat)
{
    if (I <= 0 || I > kVaeMaxItems || nh < 0 || nh > kVaeMaxHidden || lat < 2 || (nh > 0 && !hidden)) return false;
    v.I = I; v.nh = nh; v.lat = lat; v.half = lat / 2; v.ne = v.nd = nh + 1;
    v.e[0] = I;
    for (int k = 0; k < nh; ++k) {
        if (hidden[k] <= 0) return false;
        v.e[k + 1] = hidden[k];
        v.d[nh - k] = hidden[k];
    }
    v.e[nh + 1] = lat;
    v.d[0] = v.half; v.d[nh + 1] = I;
    long long off = 0;
    for (int L = 0; L < v.ne + v.nd; ++L) {
        const int *w = L < v.ne ? v.e : v.d;
        const int l = L < v.ne ? L : L - v.ne;
        v.w_off[L] = off; off += (long long)w[l] * w[l + 1];
        v.b_off[L] = off; off += w[l + 1];
    }
    v.nW = off;
    v.maxw = lat;
    for (int k = 1; k <= nh; ++k) v.maxw = v.e[k] > v.maxw ? v.e[k] : v.maxw;
    v.slices = (I + 1023) / 1024;
    if (v.slices > 16) v.slices = 16;
    return true;
}

struct VaeWs {
    WsHeader *hdr;
    float *g, *m, *v;                 // gradient / optimiser state of the flat block
    long long *boff;                  // [R + 1] batch row offsets into the nonzero scratch
    float *rs, *cerow, *klrow;        // [R] per row: sum r, CE row sum, KL row sum
    float *enc[kVaeMaxHidden + 1];    // encoder layer outputs [R, e[l+1]]
    float *z, *eps;                   // [R, half]
    float *dec[kVaeMaxHidden + 1];    // decoder layer outputs [R, d[l+1]] (the last: logits, then dz)
    float *dA, *dB;                   // [R, maxw] backward ping-pong
    float *slices;                    // [slices, R, d[nd-1]]
    int32_t *bcol;                    // [R * max_row_len] the batch's nonzeros: item
    float *bx, *br, *bz;              //           dropped normalised value, raw value, logit
    int2 *tpair;                      // [R * max_row_len] (row, nonzero) grouped by item
    unsigned *icnt, *icur;            // [I]
    long long *iptr;                  // [I + 1]
};

constexpr int kVaeOptNone = -1;              // a scoring workspace: no gradient or optimiser state

// The nonzero scratch holds R rows of max_row_len entries (the longest input row): no batch of at most R users, repeated users
// included, can outgrow it.
static size_t carve_vae(void *base, const VaeDims &d, int opt, long long R, long long max_row_len, VaeWs *w)
{
    size_t off = 0;
    char *b = (char *)base;
    auto take = [&](size_t bytes) {
        char *p = b ? b + off : nullptr;
        off += align256(bytes);
        return p;
    };
    VaeWs t;
    t.hdr = (WsHeader *)take(256);
    t.g = t.m = t.v = nullptr;
    if (opt != kVaeOptNone) t.g = (float *)take(sizeof(float) * d.nW);
    if (opt == DRB_OPT_ADAM) {
        t.m = (float *)take(sizeof(float) * d.nW);
        t.v = (float *)take(sizeof(float) * d.nW);
    }
    t.icnt = (unsigned *)take(sizeof(unsigned) * d.I);       // icnt, icur adjacent: one memset per step
    t.icur = (unsigned *)take(sizeof(unsigned) * d.I);
    t.iptr = (long long *)take(sizeof(long long) * (d.I + 1));
    t.boff = (long long *)take(sizeof(long long) * (R + 1));
    t.rs = (float *)take(sizeof(float) * R);
    t.cerow = (float *)take(sizeof(float) * R);
    t.klrow = (float *)take(sizeof(float) * R);
    for (int l = 0; l < d.ne; ++l) t.enc[l] = (float *)take(sizeof(float) * R * d.e[l + 1]);
    t.z = (float *)take(sizeof(float) * R * d.half);
    t.eps = (float *)take(sizeof(float) * R * d.half);
    for (int l = 0; l < d.nd; ++l) t.dec[l] = (float *)take(sizeof(float) * R * d.d[l + 1]);
    t.dA = (float *)take(sizeof(float) * R * d.maxw);
    t.dB = (float *)take(sizeof(float) * R * d.maxw);
    t.slices = (float *)take(sizeof(float) * d.slices * R * d.d[d.nd - 1]);
    const size_t nz = (size_t)(R * max_row_len > 0 ? R * max_row_len : 1);
    t.bcol = (int32_t *)take(sizeof(int32_t) * nz);
    t.bx = (float *)take(sizeof(float) * nz);
    t.br = (float *)take(sizeof(float) * nz);
    t.bz = (float *)take(sizeof(float) * nz);
    t.tpair = (int2 *)take(sizeof(int2) * nz);
    if (w) *w = t;
    return off;
}

__device__ __forceinline__ float warp_sum(float s)
{
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    return s;
}

// sum over a CTA of 256 threads in a fixed tree (the same partials always meet in the same order)
__device__ __forceinline__ float block_sum256(float s, float *red)
{
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    float t = 0.f;
    if (threadIdx.x < 32) {
        t = threadIdx.x < 8 ? red[threadIdx.x] : 0.f;
        t = warp_sum(t);
        if (threadIdx.x == 0) red[8] = t;
    }
    __syncthreads();
    t = red[8];
    __syncthreads();
    return t;
}

__device__ __forceinline__ float block_max256(float s, float *red)
{
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) s = fmaxf(s, __shfl_xor_sync(0xffffffffu, s, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    float t = red[0];
    for (int q = 1; q < 8; ++q) t = fmaxf(t, red[q]);
    __syncthreads();
    return t;
}

// ------------------------------------------------------------------------------------------ input CSR (once per model)
// AERecommender.get_user_rating_matrix (AbstractRecommender.py:147-158): index_put_ without accumulate, where on the CPU the last
// write of a (row, item) pair wins.  One warp per history row walks its slots from the last one back; a slot is the pair's
// effective write when no later slot names its item (a bitmap of the items already met, in shared memory).  Effective writes
// with a nonzero value are the row's entries, kept in slot order.  EMIT = false: ptr[u] = entry count.
template <bool EMIT>
__global__ void __launch_bounds__(kVaeInputThreads) vae_input_csr_kernel(const int64_t *__restrict__ hid, const float *__restrict__ hval,
                                                                         int U, int L, int I, long long *__restrict__ ptr,
                                                                         int32_t *__restrict__ col, float *__restrict__ val,
                                                                         int *__restrict__ bad)
{
    extern __shared__ uint32_t seen[];
    const int lane = threadIdx.x;
    const int words = (I + 31) >> 5;
    for (int w = lane; w < words; w += 32) seen[w] = 0u;
    __syncwarp();
    for (int u = blockIdx.x; u < U; u += gridDim.x) {
        const int64_t *ids = hid + (size_t)u * L;
        const float *vals = hval + (size_t)u * L;
        long long after = 0;                                // entries at slots above the current chunk
        const long long end = EMIT ? ptr[u + 1] : 0;
        for (int top = L - 1; top >= 0; top -= 32) {
            const int s = top - lane;
            int it = -1;
            float v = 0.f;
            if (s >= 0) {
                const int64_t raw = ids[s];
                if (raw < 0 || raw >= I) atomicOr(bad, 1);
                else { it = (int)raw; v = vals[s]; }
            }
            // among this chunk's lanes naming one item the lowest lane holds the highest slot
            const unsigned same = __match_any_sync(0xffffffffu, it);
            bool eff = it >= 0 && lane == __ffs(same) - 1 && !((seen[it >> 5] >> (it & 31)) & 1u);
            __syncwarp();
            if (it >= 0) atomicOr(&seen[it >> 5], 1u << (it & 31));
            const bool keep = eff && v != 0.f;
            const unsigned mask = __ballot_sync(0xffffffffu, keep);
            if (EMIT && keep) {
                const long long pos = end - 1 - after - __popc(mask & ((1u << lane) - 1u));
                col[pos] = it;
                val[pos] = v;
            }
            after += __popc(mask);
            __syncwarp();
        }
        if (!EMIT && lane == 0) ptr[u] = after;
        for (int s = lane; s < L; s += 32) {                // clear the row's bits for the next row
            const int64_t raw = ids[s];
            if (raw >= 0 && raw < I) seen[raw >> 5] = 0u;
        }
        __syncwarp();
    }
}

// in-place exclusive scan of n int64 counters, a[n] = total.  One CTA.
__global__ void __launch_bounds__(1024) vae_exscan_kernel(long long *__restrict__ a, long long n)
{
    __shared__ long long wtot[32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    long long carry = 0;
    for (long long base = 0; base < n; base += 1024) {
        const long long idx = base + tid;
        const long long v = idx < n ? a[idx] : 0;
        long long x = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            long long y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) wtot[warp] = x;
        __syncthreads();
        if (warp == 0) {
            long long t = wtot[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                long long y = __shfl_up_sync(0xffffffffu, t, o);
                if (lane >= o) t += y;
            }
            wtot[lane] = t;
        }
        __syncthreads();
        if (idx < n) a[idx] = carry + (warp > 0 ? wtot[warp - 1] : 0) + x - v;
        const long long total = wtot[31];
        __syncthreads();
        carry += total;
    }
    if (tid == 0) a[n] = carry;
}

__global__ void vae_widen_kernel(const unsigned *__restrict__ in, long long *__restrict__ out, int n)
{
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) out[k] = in[k];
}

// ------------------------------------------------------------------------------------------ batch input
// boff[b] = the length of user b's input row.  A row longer than the workspace's max_row_len (a workspace laid out for another
// input) is clamped, so nothing is written past the scratch, and the header's status makes the call fail.
__global__ void vae_batch_len_kernel(const int64_t *__restrict__ users, const long long *__restrict__ row_ptr, int B,
                                     long long max_row_len, long long *__restrict__ boff, WsHeader *hdr)
{
    for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < B; b += gridDim.x * blockDim.x) {
        const long long u = users[b];
        long long n = row_ptr[u + 1] - row_ptr[u];
        if (n > max_row_len) {
            n = max_row_len;
            atomicExch(&hdr->status, DRB_ERR_INVALID);
        }
        boff[b] = n;
    }
}

struct VaeDrop {
    float p, inv_keep;
    uint32_t thresh, k0, k1, step;
    const uint32_t *bits;     // host keep bits of this step, bit b * I + item; nullptr: Philox
};

__device__ __forceinline__ bool vae_keep(const VaeDrop &d, int b, int item, int I)
{
    if (d.bits) {
        const unsigned long long e = (unsigned long long)b * I + item;
        return (__ldg(d.bits + (e >> 5)) >> (e & 31)) & 1u;
    }
    uint32_t c[4] = {(uint32_t)item, (uint32_t)b, d.step, 0x56414531u};
    philox4x32(c, d.k0, d.k1);
    return c[0] >= d.thresh;
}

// the device draw of randn_like(std)[b, j] (Box-Muller on one Philox block)
__device__ __forceinline__ float vae_normal(uint32_t k0, uint32_t k1, uint32_t step, int b, int j)
{
    uint32_t c[4] = {(uint32_t)j, (uint32_t)b, step, 0x45505331u};
    philox4x32(c, k0, k1);
    const float u1 = ((c[0] >> 8) + 1) * (1.f / 16777216.f), u2 = (c[1] >> 8) * (1.f / 16777216.f);
    return sqrtf(-2.f * logf(u1)) * cospif(2.f * u2);
}

// One warp per batch row: F.normalize (:80, row L2 norm clamped at 1e-12), F.dropout (:81) at the row's nonzeros, the raw values
// for the CE and their sum.  The norm and the sum are lane-strided partials reduced in a fixed tree.
__global__ void vae_input_kernel(const int64_t *__restrict__ users, const long long *__restrict__ row_ptr,
                                 const int32_t *__restrict__ col, const float *__restrict__ val, int B, int I,
                                 const long long *__restrict__ boff, int drop_on, VaeDrop drop, int32_t *__restrict__ bcol,
                                 float *__restrict__ bx, float *__restrict__ br, float *__restrict__ rs,
                                 unsigned *__restrict__ icnt)
{
    const int lane = threadIdx.x & 31;
    const int nw = (gridDim.x * blockDim.x) >> 5;
    for (int b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; b < B; b += nw) {
        const long long u = users[b], s0 = row_ptr[u], o = boff[b], n = boff[b + 1] - o;
        float ss = 0.f, sr = 0.f;
        for (long long k = lane; k < n; k += 32) {
            const float v = val[s0 + k];
            ss = fmaf(v, v, ss);
            sr += v;
        }
        ss = warp_sum(ss);
        sr = warp_sum(sr);
        const float den = fmaxf(sqrtf(ss), 1e-12f);
        for (long long k = lane; k < n; k += 32) {
            const int it = col[s0 + k];
            const float v = val[s0 + k];
            float x = v / den;
            if (drop_on) x = vae_keep(drop, b, it, I) ? x * drop.inv_keep : 0.f;
            bcol[o + k] = it;
            bx[o + k] = x;
            br[o + k] = v;
            if (icnt) atomicAdd(icnt + it, 1u);
        }
        if (lane == 0) rs[b] = sr;
    }
}

// (row, nonzero) records grouped by item (unordered inside an item: vae_dw0_kernel orders them by row)
__global__ void vae_group_kernel(int B, const long long *__restrict__ boff, const int32_t *__restrict__ bcol,
                                 const long long *__restrict__ iptr, unsigned *__restrict__ icur, int2 *__restrict__ tpair)
{
    const int lane = threadIdx.x & 31;
    const int nw = (gridDim.x * blockDim.x) >> 5;
    for (int b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; b < B; b += nw)
        for (long long k = boff[b] + lane; k < boff[b + 1]; k += 32) {
            const int it = bcol[k];
            tpair[iptr[it] + atomicAdd(icur + it, 1u)] = make_int2(b, (int)k);
        }
}

// ------------------------------------------------------------------------------------------ encoder layer 0
// h[b, j] = act(b0[j] + sum_k x~[k] W0t[item_k, j]) over row b's nonzeros in slot order.  One CTA per row.
__global__ void __launch_bounds__(256) vae_enc0_kernel(const float *__restrict__ W0t, const float *__restrict__ b0, int H, int B,
                                                       const long long *__restrict__ boff, const int32_t *__restrict__ bcol,
                                                       const float *__restrict__ bx, int act, float *__restrict__ out)
{
    for (int b = blockIdx.x; b < B; b += gridDim.x) {
        const long long k0 = boff[b], k1 = boff[b + 1];
        for (int j = threadIdx.x; j < H; j += blockDim.x) {
            float acc = 0.f;
            for (long long k = k0; k < k1; ++k) acc = fmaf(bx[k], __ldg(W0t + (size_t)bcol[k] * H + j), acc);
            acc += b0[j];
            out[(size_t)b * H + j] = act ? tanhf(acc) : acc;
        }
    }
}

// gW0t[i, :] = sum_b x~[b, i] dZ0[b, :], rows b ascending; only the batch's items.  One CTA per item: its records are marked in
// a bitmap of the B rows, which is then walked in order.
__global__ void __launch_bounds__(256) vae_dw0_kernel(int I, int H, int B, const long long *__restrict__ iptr,
                                                      const int2 *__restrict__ tpair, const float *__restrict__ bx,
                                                      const float *__restrict__ dZ, float *__restrict__ gW0t)
{
    extern __shared__ uint32_t sm[];
    const int words = (B + 31) >> 5;
    uint32_t *bits = sm;
    int *kk = (int *)(sm + words);
    for (int i = blockIdx.x; i < I; i += gridDim.x) {
        const long long p0 = iptr[i], p1 = iptr[i + 1];
        if (p0 == p1) continue;                               // uniform across the CTA
        for (int w = threadIdx.x; w < words; w += blockDim.x) bits[w] = 0u;
        __syncthreads();
        for (long long p = p0 + threadIdx.x; p < p1; p += blockDim.x) {
            const int2 t = tpair[p];
            atomicOr(&bits[t.x >> 5], 1u << (t.x & 31));
            kk[t.x] = t.y;
        }
        __syncthreads();
        for (int j = threadIdx.x; j < H; j += blockDim.x) {
            float acc = 0.f;
            for (int w = 0; w < words; ++w) {
                uint32_t m = bits[w];
                while (m) {
                    const int b = w * 32 + __ffs(m) - 1;
                    m &= m - 1;
                    acc = fmaf(bx[kk[b]], dZ[(size_t)b * H + j], acc);
                }
            }
            gW0t[(size_t)i * H + j] = acc;
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------ dense helpers
__global__ void vae_bias_act_kernel(float *__restrict__ Z, const float *__restrict__ bias, long long M, int N, int act)
{
    const long long n = M * N;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
        const float v = Z[k] + bias[k % N];
        Z[k] = act ? tanhf(v) : v;
    }
}

// dZ *= 1 - A^2 (tanh')
__global__ void vae_tanh_back_kernel(float *__restrict__ dZ, const float *__restrict__ A, long long n)
{
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
        const float a = A[k];
        dZ[k] = dZ[k] * (1.f - a * a);
    }
}

// out = sum_z slice_z (z ascending), times 1 - A^2 when A is given
__global__ void vae_slice_sum_kernel(const float *__restrict__ sl, int S, long long n, const float *__restrict__ A,
                                     float *__restrict__ out)
{
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
        float s = sl[k];
        for (int z = 1; z < S; ++z) s += sl[(size_t)z * n + k];
        if (A) s = s * (1.f - A[k] * A[k]);
        out[k] = s;
    }
}

// gb[n] = sum_m dZ[m, n], m ascending (one thread per column; consecutive threads read consecutive columns)
__global__ void vae_colsum_kernel(const float *__restrict__ dZ, long long M, int N, float *__restrict__ gb)
{
    for (int n = blockIdx.x * blockDim.x + threadIdx.x; n < N; n += gridDim.x * blockDim.x) {
        float s = 0.f;
        for (long long m = 0; m < M; ++m) s += dZ[m * N + n];
        gb[n] = s;
    }
}

// ------------------------------------------------------------------------------------------ reparameterisation + KL
// One warp per row: mu = h[:, :half], logvar = h[:, lat - half:] (:85-86); z = eps * exp(logvar / 2) + mu in train mode, mu in
// eval mode (:71-77); klrow = sum_j (1 + logvar - mu^2 - exp(logvar)) (:102).  eps from the host (h_eps) or Philox.
__global__ void vae_reparam_kernel(const float *__restrict__ h, int B, int lat, int half, int training,
                                   const float *__restrict__ h_eps, uint32_t k0, uint32_t k1, uint32_t step,
                                   float *__restrict__ z, float *__restrict__ eps, float *__restrict__ klrow)
{
    const int lane = threadIdx.x & 31;
    const int nw = (gridDim.x * blockDim.x) >> 5;
    const int lo = lat - half;
    for (int b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; b < B; b += nw) {
        float kl = 0.f;
        for (int j = lane; j < half; j += 32) {
            const float mu = h[(size_t)b * lat + j], lv = h[(size_t)b * lat + lo + j];
            const float ev = expf(lv);
            kl += ((1.f + lv) - mu * mu) - ev;
            float e = 0.f, zz = mu;
            if (training) {
                e = h_eps ? h_eps[(size_t)b * half + j] : vae_normal(k0, k1, step, b, j);
                zz = e * expf(0.5f * lv) + mu;
            }
            z[(size_t)b * half + j] = zz;
            eps[(size_t)b * half + j] = e;
        }
        kl = warp_sum(kl);
        if (lane == 0) klrow[b] = kl;
    }
}

// dmu = dz + anneal mu / B;  dlogvar = dz eps exp(logvar / 2) / 2 + anneal (exp(logvar) - 1) / (2B);  the odd middle column 0
__global__ void vae_reparam_back_kernel(const float *__restrict__ h, const float *__restrict__ eps, const float *__restrict__ dz,
                                        int B, int lat, int half, float anneal, float *__restrict__ dh)
{
    const int lo = lat - half;
    const float invB = 1.f / (float)B;
    const long long n = (long long)B * lat;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
        const int b = (int)(k / lat), c = (int)(k % lat);
        float g = 0.f;
        if (c < half) {
            g = dz[(size_t)b * half + c] + anneal * h[k] * invB;
        } else if (c >= lo) {
            const int j = c - lo;
            const float lv = h[k];
            g = dz[(size_t)b * half + j] * eps[(size_t)b * half + j] * expf(0.5f * lv) * 0.5f + anneal * 0.5f * (expf(lv) - 1.f) * invB;
        }
        dh[k] = g;
    }
}

// ------------------------------------------------------------------------------------------ fused log-softmax cross-entropy
// One CTA per row: max, log-sum-exp, cerow = sum_k r_k log_softmax(z)[item_k] over the row's nonzeros, then the logits are
// replaced by dz = (softmax(z) sum(r) - r) / B.
__global__ void __launch_bounds__(256) vae_ce_kernel(float *__restrict__ Z, int I, int B, const long long *__restrict__ boff,
                                                     const int32_t *__restrict__ bcol, const float *__restrict__ br,
                                                     float *__restrict__ bz, const float *__restrict__ rs, int grad,
                                                     float *__restrict__ cerow)
{
    __shared__ float red[9];
    const float invB = 1.f / (float)B;
    for (int b = blockIdx.x; b < B; b += gridDim.x) {
        float *z = Z + (size_t)b * I;
        float mx = -INFINITY;
        for (int i = threadIdx.x; i < I; i += blockDim.x) mx = fmaxf(mx, z[i]);
        mx = block_max256(mx, red);
        float se = 0.f;
        for (int i = threadIdx.x; i < I; i += blockDim.x) se += expf(z[i] - mx);
        se = block_sum256(se, red);
        const float lse = logf(se);
        const long long k0 = boff[b], k1 = boff[b + 1];
        float ce = 0.f;
        for (long long k = k0 + threadIdx.x; k < k1; k += blockDim.x) {
            const float zk = z[bcol[k]];
            bz[k] = zk;
            ce = fmaf((zk - mx) - lse, br[k], ce);
        }
        ce = block_sum256(ce, red);
        if (threadIdx.x == 0) cerow[b] = ce;
        if (grad) {
            const float r = rs[b];
            for (int i = threadIdx.x; i < I; i += blockDim.x) z[i] = expf((z[i] - mx) - lse) * r * invB;
            __syncthreads();
            for (long long k = k0 + threadIdx.x; k < k1; k += blockDim.x)
                z[bcol[k]] = (expf((bz[k] - mx) - lse) * r - br[k]) * invB;
        }
        __syncthreads();
    }
}

// loss = -(sum_b cerow) / B + (-0.5 (sum_b klrow) / B) anneal (:102-105), rows summed in order; NaN -> sticky status
__global__ void vae_loss_kernel(const float *__restrict__ cerow, const float *__restrict__ klrow, int B, float anneal,
                                double *__restrict__ loss_out, WsHeader *hdr, long long step)
{
    double ce = 0.0, kl = 0.0;
    for (int b = 0; b < B; ++b) {
        ce += cerow[b];
        kl += klrow[b];
    }
    const float ce_loss = -(float)(ce / B);
    const float kl_loss = (-0.5f * (float)(kl / B)) * anneal;
    const float loss = ce_loss + kl_loss;
    *loss_out = (double)loss;
    if (isnan(loss) && hdr->status == 0) {
        hdr->status = DRB_ERR_NAN_LOSS;
        hdr->nan_step = step;
    }
}

// ------------------------------------------------------------------------------------------ scoring
// scores[r, c] = W3[cands[r, c]] . hd[r] + b3[cands[r, c]], one warp per score
__global__ void vae_score_kernel(const float *__restrict__ W3, const float *__restrict__ b3, int H, const float *__restrict__ hd,
                                 const int64_t *__restrict__ cands, long long rows, int C, float *__restrict__ out)
{
    const int lane = threadIdx.x & 31;
    const long long nw = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long q = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; q < rows * C; q += nw) {
        const long long r = q / C;
        const long long c = cands[q];
        float s = 0.f;
        for (int j = lane; j < H; j += 32) s = fmaf(W3[c * H + j], hd[r * H + j], s);
        s = warp_sum(s);
        if (lane == 0) out[q] = s + b3[c];
    }
}

// ------------------------------------------------------------------------------------------ host drivers
struct VaeInputs {
    const long long *row_ptr;
    const int32_t *col;
    const float *val;
};

// forward through the decoder's hidden layers (stops before the output layer when `to_logits` is false)
static int vae_forward(const VaeDims &d, const float *W, const VaeWs &w, const VaeInputs &in, const int64_t *users, int B,
                       long long max_row_len, int training, bool grouped, const VaeDrop &drop, int drop_on, const float *h_eps,
                       uint32_t k0, uint32_t k1, bool to_logits, cudaStream_t st)
{
    vae_batch_len_kernel<<<grid_for(B, 256), 256, 0, st>>>(users, in.row_ptr, B, max_row_len, w.boff, w.hdr);
    vae_exscan_kernel<<<1, 1024, 0, st>>>(w.boff, B);
    DRB_CUDA(cudaGetLastError());
    if (grouped) DRB_CUDA(cudaMemsetAsync(w.icnt, 0, (size_t)((char *)w.iptr - (char *)w.icnt), st));
    vae_input_kernel<<<grid_for((long long)B * 32, 256), 256, 0, st>>>(users, in.row_ptr, in.col, in.val, B, d.I, w.boff, drop_on,
                                                                      drop, w.bcol, w.bx, w.br, w.rs, grouped ? w.icnt : nullptr);
    DRB_CUDA(cudaGetLastError());
    if (grouped) {
        vae_widen_kernel<<<grid_for(d.I, 256), 256, 0, st>>>(w.icnt, w.iptr, d.I);
        vae_exscan_kernel<<<1, 1024, 0, st>>>(w.iptr, d.I);
        vae_group_kernel<<<grid_for((long long)B * 32, 256), 256, 0, st>>>(B, w.boff, w.bcol, w.iptr, w.icur, w.tpair);
        DRB_CUDA(cudaGetLastError());
    }
    vae_enc0_kernel<<<grid_for(B, 1, 8), 256, 0, st>>>(W + d.w_off[0], W + d.b_off[0], d.e[1], B, w.boff, w.bcol, w.bx,
                                                        d.ne > 1 ? 1 : 0, w.enc[0]);
    DRB_CUDA(cudaGetLastError());
    for (int l = 1; l < d.ne; ++l) {
        int rc = gemm_nt(0, B, d.e[l + 1], d.e[l], w.enc[l - 1], d.e[l], W + d.w_off[l], d.e[l], w.enc[l], d.e[l + 1], st);
        if (rc != DRB_OK) return rc;
        vae_bias_act_kernel<<<grid_for((long long)B * d.e[l + 1], 256), 256, 0, st>>>(w.enc[l], W + d.b_off[l], B, d.e[l + 1],
                                                                                      l + 1 < d.ne ? 1 : 0);
        DRB_CUDA(cudaGetLastError());
    }
    vae_reparam_kernel<<<grid_for((long long)B * 32, 256), 256, 0, st>>>(w.enc[d.ne - 1], B, d.lat, d.half, training, h_eps, k0, k1,
                                                                        drop.step, w.z, w.eps, w.klrow);
    DRB_CUDA(cudaGetLastError());
    const int last = to_logits ? d.nd : d.nd - 1;
    for (int l = 0; l < last; ++l) {
        const int L = d.ne + l;
        const float *A = l == 0 ? w.z : w.dec[l - 1];
        int rc = gemm_nt(0, B, d.d[l + 1], d.d[l], A, d.d[l], W + d.w_off[L], d.d[l], w.dec[l], d.d[l + 1], st);
        if (rc != DRB_OK) return rc;
        vae_bias_act_kernel<<<grid_for((long long)B * d.d[l + 1], 256), 256, 0, st>>>(w.dec[l], W + d.b_off[L], B, d.d[l + 1],
                                                                                      l + 1 < d.nd ? 1 : 0);
        DRB_CUDA(cudaGetLastError());
    }
    return DRB_OK;
}

// gradients of the flat block for the batch whose forward pass is in the workspace (dz already in place of the logits)
static int vae_backward(const VaeDims &d, const float *W, const VaeWs &w, int B, float anneal, cudaStream_t st)
{
    float *cur = w.dec[d.nd - 1];                             // dZ of the current layer
    float *bufs[2] = {w.dA, w.dB};
    int flip = 0;
    for (int l = d.nd - 1; l >= 0; --l) {
        const int L = d.ne + l, in = d.d[l], out = d.d[l + 1];
        const float *A = l == 0 ? w.z : w.dec[l - 1];
        int rc = gemm_tn(out, in, B, cur, out, A, in, w.g + d.w_off[L], in, st);
        if (rc != DRB_OK) return rc;
        vae_colsum_kernel<<<grid_for(out, 256), 256, 0, st>>>(cur, B, out, w.g + d.b_off[L]);
        DRB_CUDA(cudaGetLastError());
        float *nxt = bufs[flip];
        flip ^= 1;
        const float *Amask = l > 0 ? w.dec[l - 1] : nullptr;   // tanh' of the layer below (the latent z has none)
        const long long n = (long long)B * in;
        if (l == d.nd - 1 && d.slices > 1) {
            rc = gemm_nn_slices(B, in, out, cur, out, W + d.w_off[L], in, w.slices, in, d.slices, st);
            if (rc != DRB_OK) return rc;
            vae_slice_sum_kernel<<<grid_for(n, 256), 256, 0, st>>>(w.slices, d.slices, n, Amask, nxt);
        } else {
            rc = gemm_nn(0, B, in, out, cur, out, W + d.w_off[L], in, nxt, in, st);
            if (rc != DRB_OK) return rc;
            if (Amask) vae_tanh_back_kernel<<<grid_for(n, 256), 256, 0, st>>>(nxt, Amask, n);
        }
        DRB_CUDA(cudaGetLastError());
        cur = nxt;
    }
    float *dh = bufs[flip];
    flip ^= 1;
    vae_reparam_back_kernel<<<grid_for((long long)B * d.lat, 256), 256, 0, st>>>(w.enc[d.ne - 1], w.eps, cur, B, d.lat, d.half,
                                                                                 anneal, dh);
    DRB_CUDA(cudaGetLastError());
    cur = dh;
    for (int l = d.ne - 1; l >= 1; --l) {
        const int in = d.e[l], out = d.e[l + 1];
        int rc = gemm_tn(out, in, B, cur, out, w.enc[l - 1], in, w.g + d.w_off[l], in, st);
        if (rc != DRB_OK) return rc;
        vae_colsum_kernel<<<grid_for(out, 256), 256, 0, st>>>(cur, B, out, w.g + d.b_off[l]);
        DRB_CUDA(cudaGetLastError());
        float *nxt = bufs[flip];
        flip ^= 1;
        rc = gemm_nn(0, B, in, out, cur, out, W + d.w_off[l], in, nxt, in, st);
        if (rc != DRB_OK) return rc;
        vae_tanh_back_kernel<<<grid_for((long long)B * in, 256), 256, 0, st>>>(nxt, w.enc[l - 1], (long long)B * in);
        DRB_CUDA(cudaGetLastError());
        cur = nxt;
    }
    const int H = d.e[1];
    vae_colsum_kernel<<<grid_for(H, 256), 256, 0, st>>>(cur, B, H, w.g + d.b_off[0]);
    DRB_CUDA(cudaGetLastError());
    const size_t smem = sizeof(uint32_t) * ((B + 31) / 32) + sizeof(int) * (size_t)B;
    DRB_REQUIRE(smem <= kVaeDw0MaxSmem, "vae: batch %d exceeds the %d rows of the layer-0 gradient kernel", B, kVaeMaxBatch);
    vae_dw0_kernel<<<grid_for(d.I, 1, 8), 256, smem, st>>>(d.I, H, B, w.iptr, w.tpair, w.bx, cur, w.g + d.w_off[0]);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}

}  // namespace drb

using namespace drb;

// the layer-0 gradient kernel's shared memory limit, raised once per process (the attribute is per function, not per launch)
static int vae_dw0_smem_once()
{
    static int rc = [] {
        return cudaFuncSetAttribute(vae_dw0_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kVaeDw0MaxSmem) == cudaSuccess
                   ? DRB_OK : DRB_ERR_CUDA;
    }();
    return rc;
}

// gradient block left over from a step whose loss was NaN (dense_update skipped it and did not clear it): zeroed before the
// next call's steps, so no stale row is applied later
__global__ void vae_clear_stale_kernel(float *__restrict__ g, long long n, const WsHeader *hdr)
{
    if (hdr->status == 0) return;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) g[k] = 0.f;
}

// the status a call's kernels left in the header: DRB_ERR_INVALID when an input row outgrew the workspace (synchronises)
static int vae_check_status(const WsHeader *hdr, cudaStream_t st, int64_t *nan_step)
{
    int status = 0;
    DRB_CUDA(cudaMemcpyAsync(&status, &hdr->status, sizeof(int), cudaMemcpyDeviceToHost, st));
    DRB_CUDA(cudaStreamSynchronize(st));
    DRB_REQUIRE(status != DRB_ERR_INVALID, "vae: an input row is longer than the workspace's max_row_len");
    return check_nan((void *)hdr, st, nan_step);
}

extern "C" int64_t drb_vae_param_count(int32_t item_num, const int32_t *h_hidden, int32_t n_hidden, int32_t latent_dim)
{
    VaeDims d;
    if (!vae_dims(d, item_num, h_hidden, n_hidden, latent_dim)) return -1;
    return d.nW;
}

extern "C" size_t drb_vae_workspace_bytes(int32_t item_num, const int32_t *h_hidden, int32_t n_hidden, int32_t latent_dim,
                                          int32_t opt, int64_t max_rows, int32_t max_row_len)
{
    VaeDims d;
    if (!vae_dims(d, item_num, h_hidden, n_hidden, latent_dim) || max_rows <= 0 || max_rows > kVaeMaxBatch || max_row_len < 0) return 0;
    return carve_vae(nullptr, d, opt, max_rows, max_row_len, nullptr);
}

extern "C" int drb_vae_workspace_init(void *d_ws, int32_t item_num, const int32_t *h_hidden, int32_t n_hidden,
                                      int32_t latent_dim, int32_t opt, int64_t max_rows, int32_t max_row_len, void *stream)
{
    VaeDims d;
    DRB_REQUIRE(d_ws && vae_dims(d, item_num, h_hidden, n_hidden, latent_dim) && max_rows > 0 && max_rows <= kVaeMaxBatch && max_row_len >= 0,
                "vae_workspace_init: bad arguments");
    VaeWs w;
    carve_vae(d_ws, d, opt, max_rows, max_row_len, &w);
    // header, gradient and optimiser state; the scratch after them is written before it is read
    DRB_CUDA(cudaMemsetAsync(d_ws, 0, (size_t)((char *)w.icnt - (char *)d_ws), (cudaStream_t)stream));
    return vae_dw0_smem_once();
}

extern "C" int drb_vae_input_csr(const int64_t *d_hist_id, const float *d_hist_val, int32_t user_num, int32_t max_len,
                                 int32_t item_num, int64_t *d_row_ptr, int32_t *d_col, float *d_val, int64_t *h_nnz, void *stream)
{
    DRB_REQUIRE(d_row_ptr && h_nnz && user_num > 0 && max_len >= 0 && item_num > 0 && (max_len == 0 || (d_hist_id && d_hist_val)),
                "vae_input_csr: bad arguments");
    DRB_REQUIRE(item_num <= kVaeMaxItems, "vae_input_csr: item_num %d exceeds %d", item_num, kVaeMaxItems);
    cudaStream_t st = (cudaStream_t)stream;
    const size_t smem = sizeof(uint32_t) * (size_t)((item_num + 31) / 32);
    if (smem > 48 * 1024) {
        DRB_CUDA(cudaFuncSetAttribute(vae_input_csr_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        DRB_CUDA(cudaFuncSetAttribute(vae_input_csr_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    int *bad = nullptr;
    DRB_CUDA(cudaMallocAsync((void **)&bad, sizeof(int), st));
    DRB_CUDA(cudaMemsetAsync(bad, 0, sizeof(int), st));
    long long *ptr = (long long *)d_row_ptr;
    const int grid = grid_for(user_num, 1, smem > 32 * 1024 ? 2 : 16);
    if (d_col == nullptr) {   // count: d_row_ptr = the exclusive scan of the entry counts, *h_nnz = the total
        vae_input_csr_kernel<false><<<grid, kVaeInputThreads, smem, st>>>(d_hist_id, d_hist_val, user_num, max_len, item_num, ptr,
                                                                        nullptr, nullptr, bad);
        vae_exscan_kernel<<<1, 1024, 0, st>>>(ptr, user_num);
    } else {                  // emit into the arrays sized by the count call
        DRB_REQUIRE(d_val, "vae_input_csr: null d_val");
        vae_input_csr_kernel<true><<<grid, kVaeInputThreads, smem, st>>>(d_hist_id, d_hist_val, user_num, max_len, item_num, ptr,
                                                                       d_col, d_val, bad);
    }
    DRB_CUDA(cudaGetLastError());
    int h_bad = 0;
    DRB_CUDA(cudaMemcpyAsync(&h_bad, bad, sizeof(int), cudaMemcpyDeviceToHost, st));
    DRB_CUDA(cudaMemcpyAsync(h_nnz, d_row_ptr + user_num, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    DRB_CUDA(cudaFreeAsync(bad, st));
    DRB_CUDA(cudaStreamSynchronize(st));
    DRB_REQUIRE(h_bad == 0, "vae_input_csr: a history item id lies outside [0, %d)", item_num);
    return DRB_OK;
}

static VaeDrop make_drop(float dropout, uint64_t seed, long long step, const uint32_t *bits)
{
    VaeDrop dr;
    dr.p = dropout;
    dr.inv_keep = 1.f / (float)(1.0 - (double)dropout);
    dr.thresh = (uint32_t)fmin(4294967295.0, (double)dropout * 4294967296.0);
    dr.k0 = (uint32_t)seed;
    dr.k1 = (uint32_t)(seed >> 32);
    dr.step = (uint32_t)step;
    dr.bits = bits;
    return dr;
}

extern "C" int drb_vae_train_steps(float *d_W, void *d_ws, int32_t item_num, const int32_t *h_hidden, int32_t n_hidden,
                                   int32_t latent_dim, int32_t opt, int64_t max_rows, int32_t max_row_len, const int64_t *d_row_ptr,
                                   const int32_t *d_col, const float *d_val, const int64_t *d_users, int64_t n, int64_t batch,
                                   int64_t first_step, int64_t n_steps, const drb_hyper *hyper, int64_t adam_step0, int32_t apply,
                                   int32_t training, int64_t update0, int64_t total_anneal_steps, double anneal_cap,
                                   float dropout, uint64_t seed, const uint32_t *d_keep_bits, const float *d_eps,
                                   double *d_step_loss, int32_t sync_and_check, int64_t *nan_step, void *stream)
{
    VaeDims d;
    DRB_REQUIRE(vae_dims(d, item_num, h_hidden, n_hidden, latent_dim), "vae: bad dims (1 <= item_num <= %d, latent_dim >= 2)",
                kVaeMaxItems);
    DRB_REQUIRE(d_W && d_ws && d_row_ptr && d_users && hyper && d_step_loss && batch > 0 && batch <= max_rows,
                "vae_train_steps: bad arguments (batch %lld, max_rows %lld)", (long long)batch, (long long)max_rows);
    DRB_REQUIRE(dropout >= 0.f && dropout < 1.f, "vae: dropout must be in [0, 1)");
    DRB_REQUIRE(hyper->opt == DRB_OPT_SGD || hyper->opt == DRB_OPT_ADAM, "vae: optimizer id %d (sgd / adam only)", hyper->opt);
    DRB_REQUIRE(hyper->opt == opt, "vae: the workspace was laid out for optimizer %d", opt);
    DRB_REQUIRE(n_steps == 0 || (first_step + n_steps - 1) * batch < n, "vae: steps exceed %lld rows", (long long)n);
    if (n_steps == 0) return DRB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    VaeWs w;
    carve_vae(d_ws, d, opt, max_rows, max_row_len, &w);
    VaeInputs in{(const long long *)d_row_ptr, d_col, d_val};
    if (apply) {
        vae_clear_stale_kernel<<<grid_for(d.nW, 256), 256, 0, st>>>(w.g, d.nW, w.hdr);
        DRB_CUDA(cudaGetLastError());
    }
    DRB_CUDA(cudaMemsetAsync(w.hdr, 0, sizeof(WsHeader), st));
    for (int64_t s = 0; s < n_steps; ++s) {
        const int64_t base = (first_step + s) * batch, B = (n - base < batch) ? n - base : batch;
        if (d_keep_bits || d_eps)
            DRB_REQUIRE(B == batch, "vae: host masks and eps need full batches (one call per ragged batch)");
        const long long upd = update0 + s + 1;
        const double a = total_anneal_steps > 0 ? fmin(anneal_cap, (double)upd / (double)total_anneal_steps) : anneal_cap;
        const float anneal = (float)a;
        const long long mask_words = ((long long)batch * item_num + 31) / 32;
        const bool drop_on = training && dropout > 0.f;
        VaeDrop drop = make_drop(dropout, seed, adam_step0 + s, d_keep_bits ? d_keep_bits + s * mask_words : nullptr);
        const float *h_eps = d_eps ? d_eps + s * batch * d.half : nullptr;
        int rc = vae_forward(d, d_W, w, in, d_users + base, (int)B, max_row_len, training, apply != 0, drop, drop_on ? 1 : 0, h_eps,
                             drop.k0, drop.k1, true, st);
        if (rc != DRB_OK) return rc;
        vae_ce_kernel<<<grid_for(B, 1, 8), 256, 0, st>>>(w.dec[d.nd - 1], d.I, (int)B, w.boff, w.bcol, w.br, w.bz, w.rs,
                                                          apply ? 1 : 0, w.cerow);
        vae_loss_kernel<<<1, 1, 0, st>>>(w.cerow, w.klrow, (int)B, anneal, d_step_loss + s, w.hdr, first_step + s);
        DRB_CUDA(cudaGetLastError());
        if (!apply) break;
        rc = vae_backward(d, d_W, w, (int)B, anneal, st);
        if (rc == DRB_OK) rc = dense_update(d_W, w.g, w.m, w.v, d.nW, hyper, adam_step0 + s, w.hdr, st);
        if (rc != DRB_OK) return rc;
    }
    if (sync_and_check) return vae_check_status(w.hdr, st, nan_step);
    return DRB_OK;
}

extern "C" int drb_vae_scores(const float *d_W, void *d_ws, int32_t item_num, const int32_t *h_hidden, int32_t n_hidden,
                              int32_t latent_dim, int32_t opt, int64_t max_rows, int32_t max_row_len, const int64_t *d_row_ptr,
                              const int32_t *d_col, const float *d_val, const int64_t *d_users, int64_t n_users,
                              const int64_t *d_cands, int32_t cand_num, float *d_scores, void *stream)
{
    VaeDims d;
    DRB_REQUIRE(vae_dims(d, item_num, h_hidden, n_hidden, latent_dim), "vae_scores: bad dims");
    DRB_REQUIRE(d_W && d_ws && d_row_ptr && d_users && d_scores && max_rows > 0 && n_users >= 0 &&
                    (d_cands ? cand_num > 0 : cand_num == item_num),
                "vae_scores: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    VaeWs w;
    carve_vae(d_ws, d, opt, max_rows, max_row_len, &w);
    VaeInputs in{(const long long *)d_row_ptr, d_col, d_val};
    const VaeDrop drop = make_drop(0.f, 0, 0, nullptr);
    DRB_CUDA(cudaMemsetAsync(w.hdr, 0, sizeof(WsHeader), st));
    const int Lo = d.ne + d.nd - 1, H = d.d[d.nd - 1];
    for (long long r0 = 0; r0 < n_users; r0 += max_rows) {
        const int R = (int)(n_users - r0 < max_rows ? n_users - r0 : max_rows);
        int rc = vae_forward(d, d_W, w, in, d_users + r0, R, max_row_len, 0, false, drop, 0, nullptr, 0, 0, false, st);
        if (rc != DRB_OK) return rc;
        const float *hd = d.nd > 1 ? w.dec[d.nd - 2] : w.z;
        if (d_cands) {
            vae_score_kernel<<<grid_for((long long)R * cand_num * 32, 256), 256, 0, st>>>(
                d_W + d.w_off[Lo], d_W + d.b_off[Lo], H, hd, d_cands + r0 * cand_num, R, cand_num, d_scores + r0 * cand_num);
        } else {
            float *out = d_scores + r0 * item_num;
            rc = gemm_nt(0, R, item_num, H, hd, H, d_W + d.w_off[Lo], H, out, item_num, st);
            if (rc != DRB_OK) return rc;
            vae_bias_act_kernel<<<grid_for((long long)R * item_num, 256), 256, 0, st>>>(out, d_W + d.b_off[Lo], R, item_num, 0);
        }
        DRB_CUDA(cudaGetLastError());
    }
    return vae_check_status(w.hdr, st, nullptr);
}

__global__ void vae_draws_kernel(VaeDrop drop, int rows, int cols, int half, uint8_t *__restrict__ keep, float *__restrict__ eps)
{
    const long long nk = (long long)rows * cols, n = nk + (long long)rows * half;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
        if (k < nk) keep[k] = vae_keep(drop, (int)(k / cols), (int)(k % cols), cols) ? 1 : 0;
        else eps[k - nk] = vae_normal(drop.k0, drop.k1, drop.step, (int)((k - nk) / half), (int)((k - nk) % half));
    }
}

// Test hook: the 'philox' engine's keep bits of a [rows, cols] batch and its normals [rows, half] at one step, from the very
// device functions the step uses (vae_keep, vae_normal)
extern "C" int drb_vae_philox_draws(uint64_t seed, int64_t step, float dropout, int32_t rows, int32_t cols, int32_t half,
                                    uint8_t *d_keep, float *d_eps, void *stream)
{
    DRB_REQUIRE(d_keep && d_eps && rows > 0 && cols > 0 && half > 0 && dropout >= 0.f && dropout < 1.f,
                "vae_philox_draws: bad arguments");
    const VaeDrop drop = make_drop(dropout, seed, step, nullptr);
    vae_draws_kernel<<<grid_for((long long)rows * (cols + half), 256), 256, 0, (cudaStream_t)stream>>>(drop, rows, cols, half,
                                                                                                      d_keep, d_eps);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}
