// skipgram.cu -- the skip-gram negative sampler of Item2Vec on the device.
//
// Stands behind SkipGramNegativeSampler.sampling() (daisy/utils/sampler.py:105-160).  The reference groups the train rows
// into one item sequence per user (groupby(user)[item].agg(list): users ascending, each user's items in row order, duplicates
// kept) and walks every sequence position i of a sequence of length L in Python:
//   rows (target, seq[j], 1) for the contexts j = max(0, i-w) .. min(L-1, i+w), j != i, ascending, then
//   c_i rows (target, neg, 0), neg = np.random.choice(setdiff1d(arange(I), train_ur[u]), size=c_i), c_i = #contexts.
// Here:
//   drb_skipgram_group        count rows per user -> exclusive scans (sequence offsets, and context offsets from the closed
//                             form of sum_i c_i) -> scatter row ids into their user's segment -> sort each segment's row ids
//                             (restores row order: the grouping is stable) -- all on the device;
//   drb_skipgram_draws_mt19937 (sampler.cu) the c_i bounded MT19937 draws per position, sequential on the host;
//   drb_skipgram_emit         one thread per sequence position writes its 2 c_i rows at their final offset; each negative is
//                             the k-th item outside the user's sorted train row (the binary search of kth_complement_kernel).
#include "common.cuh"

namespace drb {

constexpr int kSgSortMax = 16384;   // segments up to this length are sorted in shared memory (64 KiB)

// number of contexts of position i in a sequence of length L with window w
__host__ __device__ __forceinline__ long long sg_ctx(long long i, long long L, long long w)
{
    const long long lo = i - w > 0 ? i - w : 0, hi = i + w < L - 1 ? i + w : L - 1;
    return hi - lo;
}

// sum of sg_ctx(j, L, w) over j < i (closed form; i = L gives the sequence's total)
__host__ __device__ __forceinline__ long long sg_ctx_prefix(long long i, long long L, long long w)
{
    // sum_{j<i} min(L-1, j+w): the first a terms are j + w, the rest L - 1
    long long a = L - w > 0 ? L - w : 0;
    if (a > i) a = i;
    const long long s1 = a * (a - 1) / 2 + a * w + (i - a) * (L - 1);
    // sum_{j<i} max(0, j-w) = 1 + 2 + ... + b
    const long long b = i - w - 1 > 0 ? i - w - 1 : 0;
    return s1 - b * (b + 1) / 2;
}

__global__ void sg_count_kernel(const int32_t *__restrict__ coo_u, long long n, int U, unsigned *__restrict__ cnt,
                                int *__restrict__ bad)
{
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
        const int u = __ldg(coo_u + k);
        if (u < 0 || u >= U) { *bad = 1; continue; }
        atomicAdd(cnt + u, 1u);
    }
}

// per user: sequence length and total number of contexts
__global__ void sg_lengths_kernel(const unsigned *__restrict__ cnt, int U, int w, int64_t *__restrict__ len,
                                  int64_t *__restrict__ ctx)
{
    for (long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x; u < U; u += (long long)gridDim.x * blockDim.x) {
        const long long L = cnt[u];
        len[u] = L;
        ctx[u] = L > 0 ? sg_ctx_prefix(L, L, w) : 0;
    }
}

// exclusive scan of n int64 values, out[n] = total.  One CTA: n is a user count.
__global__ void __launch_bounds__(1024) sg_exscan_kernel(const int64_t *__restrict__ in, int64_t *__restrict__ out, long long n)
{
    __shared__ long long wtot[32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    long long carry = 0;
    for (long long base = 0; base < n; base += 1024) {
        const long long idx = base + tid;
        const long long v = idx < n ? (long long)in[idx] : 0;
        long long x = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const long long y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) wtot[warp] = x;
        __syncthreads();
        if (warp == 0) {
            long long t = wtot[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const long long y = __shfl_up_sync(0xffffffffu, t, o);
                if (lane >= o) t += y;
            }
            wtot[lane] = t;
        }
        __syncthreads();
        if (idx < n) out[idx] = carry + (warp > 0 ? wtot[warp - 1] : 0) + x - v;
        const long long total = wtot[31];
        __syncthreads();
        carry += total;
    }
    if (tid == 0) out[n] = carry;
}

__global__ void sg_scatter_kernel(const int32_t *__restrict__ coo_u, long long n, int U, const int64_t *__restrict__ seq_ptr,
                                  unsigned *__restrict__ cursor, int32_t *__restrict__ order)
{
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
        const int u = __ldg(coo_u + k);
        if (u < 0 || u >= U) continue;
        order[seq_ptr[u] + atomicAdd(cursor + u, 1u)] = (int32_t)k;
    }
}

// One CTA per user (grid-stride): sort the row ids of the user's segment ascending.  Segments up to kSgSortMax: bitonic sort
// in shared memory; longer ones: each id's rank is counted over the segment and the ids are placed through `tmp`.
__global__ void __launch_bounds__(256) sg_segsort_kernel(const int64_t *__restrict__ seq_ptr, int U, int32_t *__restrict__ order,
                                                         int32_t *__restrict__ tmp)
{
    extern __shared__ int32_t s_key[];
    const int tid = threadIdx.x;
    for (int u = blockIdx.x; u < U; u += gridDim.x) {
        const long long b = seq_ptr[u], L = seq_ptr[u + 1] - b;
        if (L < 2) continue;   // uniform across the CTA
        int32_t *seg = order + b;
        if (L <= kSgSortMax) {
            int P = 2;
            while (P < L) P <<= 1;
            for (int t = tid; t < P; t += blockDim.x) s_key[t] = t < L ? seg[t] : INT32_MAX;
            __syncthreads();
            for (int k = 2; k <= P; k <<= 1)
                for (int j = k >> 1; j > 0; j >>= 1) {
                    for (int t = tid; t < P; t += blockDim.x) {
                        const int o = t ^ j;
                        if (o > t) {
                            const int32_t x = s_key[t], y = s_key[o];
                            if ((x > y) == ((t & k) == 0)) { s_key[t] = y; s_key[o] = x; }
                        }
                    }
                    __syncthreads();
                }
            for (int t = tid; t < L; t += blockDim.x) seg[t] = s_key[t];
        } else {
            for (long long p = tid; p < L; p += blockDim.x) {
                const int32_t v = seg[p];
                long long r = 0;
                for (long long q = 0; q < L; ++q) r += seg[q] < v;
                tmp[b + r] = v;
            }
            __syncthreads();
            for (long long p = tid; p < L; p += blockDim.x) seg[p] = tmp[b + p];
        }
        __syncthreads();
    }
}

// One thread per grouped position k: user u (row order[k]), position i = k - seq_ptr[u] of a sequence of length L.
// Its 2 c_i rows start at 2 (ctx_ptr[u] + sg_ctx_prefix(i)); its draws at ctx_ptr[u] + sg_ctx_prefix(i).
__global__ void sg_emit_kernel(const int32_t *__restrict__ coo_u, const int32_t *__restrict__ coo_i,
                               const int32_t *__restrict__ order, long long n, int w, const int64_t *__restrict__ seq_ptr,
                               const int64_t *__restrict__ ctx_ptr, const int64_t *__restrict__ row_ptr,
                               const int32_t *__restrict__ col, const int32_t *__restrict__ draws, int32_t *__restrict__ rows)
{
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
        const int32_t r = __ldg(order + k);
        const int u = __ldg(coo_u + r);
        const int target = __ldg(coo_i + r);
        const long long sb = seq_ptr[u], L = seq_ptr[u + 1] - sb, i = k - sb;
        const long long c = sg_ctx(i, L, w);
        if (c == 0) continue;
        const long long d0 = ctx_ptr[u] + sg_ctx_prefix(i, L, w);
        int32_t *out = rows + 3 * (2 * d0);
        const long long lo = i - w > 0 ? i - w : 0, hi = i + w < L - 1 ? i + w : L - 1;
        for (long long j = lo; j <= hi; ++j) {
            if (j == i) continue;
            out[0] = target;
            out[1] = __ldg(coo_i + __ldg(order + sb + j));
            out[2] = 1;
            out += 3;
        }
        const long long rb = row_ptr[u], re = row_ptr[u + 1];
        for (long long m = 0; m < c; ++m) {
            const int kk = __ldg(draws + d0 + m);
            long long a = 0, z = re - rb;   // first s with col[s] - s > k: item = k + s
            while (a < z) {
                const long long mid = (a + z) >> 1;
                if ((long long)__ldg(col + rb + mid) - mid <= (long long)kk) a = mid + 1; else z = mid;
            }
            out[0] = target;
            out[1] = kk + (int)a;
            out[2] = 0;
            out += 3;
        }
    }
}

struct SgWs {
    int *bad;
    unsigned *cnt, *cursor;
    int64_t *len, *ctx;
    int32_t *tmp;
};

static size_t carve_sg(void *base, int U, long long n, SgWs *w)
{
    size_t off = 0;
    char *b = (char *)base;
    auto take = [&](size_t bytes) {
        char *p = b ? b + off : nullptr;
        off += (bytes + 255) & ~(size_t)255;
        return p;
    };
    SgWs t;
    t.bad = (int *)take(256);
    t.cnt = (unsigned *)take(sizeof(unsigned) * (size_t)U);
    t.cursor = (unsigned *)take(sizeof(unsigned) * (size_t)U);
    t.len = (int64_t *)take(sizeof(int64_t) * (size_t)U);
    t.ctx = (int64_t *)take(sizeof(int64_t) * (size_t)U);
    t.tmp = (int32_t *)take(sizeof(int32_t) * (size_t)(n > 0 ? n : 1));
    if (w) *w = t;
    return off;
}

}  // namespace drb

using namespace drb;

extern "C" size_t drb_skipgram_workspace_bytes(int32_t user_num, int64_t nnz)
{
    if (user_num <= 0 || nnz < 0) return 0;
    return carve_sg(nullptr, user_num, nnz, nullptr);
}

extern "C" int drb_skipgram_group(const int32_t *d_coo_u, int64_t nnz, int32_t user_num, int32_t window, void *d_ws,
                                  int64_t *d_seq_ptr, int64_t *d_ctx_ptr, int32_t *d_order, void *stream)
{
    DRB_REQUIRE(d_ws && d_seq_ptr && d_ctx_ptr && user_num > 0 && nnz >= 0 && window >= 0 && (nnz == 0 || (d_coo_u && d_order)),
                "skipgram_group: bad arguments");
    DRB_REQUIRE(nnz < (1LL << 31), "skipgram_group: %lld rows exceed int32 row ids", (long long)nnz);
    cudaStream_t st = (cudaStream_t)stream;
    SgWs w;
    carve_sg(d_ws, user_num, nnz, &w);
    DRB_CUDA(cudaMemsetAsync(d_ws, 0, (size_t)((char *)w.len - (char *)d_ws), st));   // bad flag, counts, cursors
    if (nnz) sg_count_kernel<<<grid_for(nnz, 256), 256, 0, st>>>(d_coo_u, nnz, user_num, w.cnt, w.bad);
    sg_lengths_kernel<<<grid_for(user_num, 256), 256, 0, st>>>(w.cnt, user_num, window, w.len, w.ctx);
    sg_exscan_kernel<<<1, 1024, 0, st>>>(w.len, d_seq_ptr, user_num);
    sg_exscan_kernel<<<1, 1024, 0, st>>>(w.ctx, d_ctx_ptr, user_num);
    if (nnz) {
        sg_scatter_kernel<<<grid_for(nnz, 256), 256, 0, st>>>(d_coo_u, nnz, user_num, d_seq_ptr, w.cursor, d_order);
        const size_t smem = sizeof(int32_t) * kSgSortMax;
        DRB_CUDA(cudaFuncSetAttribute(sg_segsort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        sg_segsort_kernel<<<grid_for(user_num, 1, 3), 256, smem, st>>>(d_seq_ptr, user_num, d_order, w.tmp);
    }
    DRB_CUDA(cudaGetLastError());
    int bad = 0;
    DRB_CUDA(cudaMemcpyAsync(&bad, w.bad, sizeof(int), cudaMemcpyDeviceToHost, st));
    DRB_CUDA(cudaStreamSynchronize(st));
    DRB_REQUIRE(bad == 0, "skipgram_group: a user id lies outside [0, %d)", user_num);
    return DRB_OK;
}

extern "C" int drb_skipgram_emit(const int32_t *d_coo_u, const int32_t *d_coo_i, const int32_t *d_order, int64_t nnz,
                                 int32_t window, const int64_t *d_seq_ptr, const int64_t *d_ctx_ptr, const int64_t *d_row_ptr,
                                 const int32_t *d_col, const int32_t *d_draws, int32_t *d_rows, void *stream)
{
    DRB_REQUIRE(d_seq_ptr && d_ctx_ptr && d_row_ptr && nnz >= 0 && window >= 0, "skipgram_emit: bad arguments");
    if (nnz == 0) return DRB_OK;
    DRB_REQUIRE(d_coo_u && d_coo_i && d_order, "skipgram_emit: null arrays");
    sg_emit_kernel<<<grid_for(nnz, 256), 256, 0, (cudaStream_t)stream>>>(d_coo_u, d_coo_i, d_order, nnz, window, d_seq_ptr,
                                                                         d_ctx_ptr, d_row_ptr, d_col, d_draws, d_rows);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}
