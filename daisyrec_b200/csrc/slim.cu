// slim.cu -- SLiM (daisy/model/SLiMRecommender.py, Ning & Karypis 2011) on the device.
//
// The reference fits one sklearn ElasticNet(positive, no intercept) per item j against y = X[:, j] with column j zeroed.  In
// Gram form, with G = X^T X (ease.cu's exact / DMMA Gram), q = G[:, j] (q_j = 0), l1 = alpha elastic U, l2 = alpha (1 -
// elastic) U, each fit is
//     min_{w >= 0, w_j = 0}  1/2 w^T G w - q^T w + l1 sum(w) + 1/2 l2 |w|^2,
// strongly convex (l2 > 0), so its optimum is unique; the reference's random coordinate order only changes the path to it.
//
//   slim_live_kernel    per target j the coordinates that can ever be non-zero, by ascending id.  With X >= 0, G >= 0 and
//                       G w >= 0, so Z = q - G w <= q along the whole iteration and a coordinate with q_k <= l1 never leaves 0:
//                       it is dead.  Dead coordinates do not move the gap either (their X^T A_k = Z_k <= l1 never decides the
//                       dual norm's comparison with l1, their w_k is 0).  With negative values, or when asked, every coordinate
//                       with G_kk > 0 is live.  The test uses a margin of 2^-20 l1 so rounding in Z can never wake a dead one.
//   slim_solve_kernel   a warp per target: cyclic coordinate descent over the live list,
//                       w_k <- max(Z_k + G_kk w_k - l1, 0) / (G_kk + l2), Z -= d G[k, live] when w_k moved;
//                       sklearn's checks (_cd_fast.pyx sparse_enet_coordinate_descent): the formulation-A duality gap before
//                       the first sweep and after every sweep with w_max == 0, d_w_max / w_max <= tol, or the last one; stop
//                       at gap <= tol G_jj.  The gap's sums run left to right over the live list and skip w_k == 0 terms
//                       exactly, so a fit with every coordinate live is bitwise the fit with the live list.  No atomics.
//   slim_select_kernel  a CTA per target: nnz = #{w_k > 0}, keep the min(nnz - 1, topk) largest by (value descending, id
//                       ascending) -- the reference's local_topk, which drops the smallest non-zero coefficient when
//                       nnz <= topk -- rounded to fp32 and stored by ascending id in itemknn.cu's neighbour layout.
#include "common.cuh"

namespace drb {

constexpr int kSlimThreads = 256;
constexpr int kSlimSolveWarps = 4;

struct SlimParams {
    double l1, l2, tol;
    int max_iter;
};

// position of this thread's flag among the CTA's set flags (thread order), and their number
__device__ __forceinline__ int slim_flag_rank(bool flag, int *s_warp, int &total)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned bal = __ballot_sync(0xffffffffu, flag);
    if (lane == 0) s_warp[warp] = __popc(bal);
    __syncthreads();
    int before = 0, all = 0;
#pragma unroll
    for (int w = 0; w < kSlimThreads / 32; ++w) {
        const int c = s_warp[w];
        before += w < warp ? c : 0;
        all += c;
    }
    __syncthreads();
    total = all;
    return before + __popc(bal & ((1u << lane) - 1u));
}

__device__ __forceinline__ int slim_block_sum(int v, int *s_warp)
{
    v = __reduce_add_sync(0xffffffffu, v);
    if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = v;
    __syncthreads();
    int all = 0;
#pragma unroll
    for (int w = 0; w < kSlimThreads / 32; ++w) all += s_warp[w];
    __syncthreads();
    return all;
}

__global__ void slim_diag_kernel(const double *__restrict__ G, int n, double *__restrict__ diag)
{
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x)
        diag[k] = G[k * n + k];
}

// one CTA per target r of the panel (item j = begin + r): the live list, w = 0 and Z = q on it
__global__ void __launch_bounds__(kSlimThreads) slim_live_kernel(const double *__restrict__ G, const double *__restrict__ diag, int n,
                                                                 int begin, double thr, int all_live, int32_t *__restrict__ lidx,
                                                                 double *__restrict__ w, double *__restrict__ z,
                                                                 int32_t *__restrict__ nl)
{
    __shared__ int s_warp[kSlimThreads / 32];
    const int r = blockIdx.x, j = begin + r, tid = threadIdx.x;
    const double *row = G + (long long)j * n;   // G is symmetric: row j holds q
    const long long base = (long long)r * n;
    int count = 0;
    for (int k0 = 0; k0 < n; k0 += kSlimThreads) {
        const int k = k0 + tid;
        double q = 0.0;
        bool live = false;
        if (k < n && k != j) {
            q = row[k];
            live = diag[k] > 0.0 && (all_live || q > thr);
        }
        int total;
        const int pos = slim_flag_rank(live, s_warp, total);
        if (live) {
            lidx[base + count + pos] = k;
            w[base + count + pos] = 0.0;
            z[base + count + pos] = q;
        }
        count += total;
    }
    if (tid == 0) nl[r] = count;
}

// acc + term of lane 0 + term of lane 1 + ... in that order (every lane returns the same sum)
__device__ __forceinline__ double slim_ordered_add(double acc, double term)
{
#pragma unroll
    for (int l = 0; l < 32; ++l) acc = __dadd_rn(acc, __shfl_sync(0xffffffffu, term, l));
    return acc;
}

// formulation-A duality gap (_cd_fast.pyx gap_enet_sparse / dual_gap_formulation_A) from w, Z = q - G w and q on the live
// list; yy = y.y = G_jj.  R.R = yy - 2 w.q + w.Gw, R.y = yy - w.q, X^T A = Z - l2 w (0 on the dead, empty and own columns).
__device__ __forceinline__ double slim_gap(const double *qrow, const int32_t *li, const double *wr, const double *zr, int cnt, double yy,
                           const SlimParams p)
{
    const int lane = threadIdx.x & 31;
    double wq = 0.0, wgw = 0.0, l1n = 0.0, l2n = 0.0, dmax = 0.0;
    for (int p0 = 0; p0 < cnt; p0 += 32) {
        const int t = p0 + lane;
        double wk = 0.0, a = 0.0, b = 0.0;
        if (t < cnt) {
            const double zk = zr[t];
            wk = wr[t];
            dmax = fmax(dmax, __dsub_rn(zk, __dmul_rn(p.l2, wk)));
            if (wk != 0.0) {
                const double q = qrow[li[t]];
                a = __dmul_rn(wk, q);
                b = __dmul_rn(wk, __dsub_rn(q, zk));
            }
        }
        if (__ballot_sync(0xffffffffu, wk != 0.0) == 0u) continue;   // every term 0: adding them changes no sum
        wq = slim_ordered_add(wq, a);
        wgw = slim_ordered_add(wgw, b);
        l1n = slim_ordered_add(l1n, wk);
        l2n = slim_ordered_add(l2n, __dmul_rn(wk, wk));
    }
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) dmax = fmax(dmax, __shfl_xor_sync(0xffffffffu, dmax, off));
    const double r2 = __dadd_rn(__dsub_rn(yy, __dmul_rn(2.0, wq)), wgw);
    const double ry = __dsub_rn(yy, wq);
    const double quad = __dadd_rn(r2, __dmul_rn(p.l2, l2n));
    const double primal = __dadd_rn(__dmul_rn(0.5, quad), __dmul_rn(p.l1, l1n));
    const double scale = dmax > p.l1 ? __ddiv_rn(p.l1, dmax) : 1.0;
    const double dual = __dadd_rn(__dmul_rn(__dmul_rn(-0.5, __dmul_rn(scale, scale)), quad), __dmul_rn(scale, ry));
    return __dsub_rn(primal, dual);
}

// a warp per target.  A live list of at most kSlimLocal coordinates (most targets) is staged in shared memory with its
// G_kk, so a coordinate update waits on shared memory and the row gather G[k, live] only; longer lists stay in global memory.
// w and z are read back by other lanes after __syncwarp, so they are not __restrict__.
constexpr int kSlimLocal = 256;

__global__ void __launch_bounds__(kSlimSolveWarps * 32) slim_solve_kernel(const double *__restrict__ G, const double *__restrict__ diag,
                                                                          int n, int begin, int count, const SlimParams p,
                                                                          const int32_t *__restrict__ lidx, double *w, double *z,
                                                                          const int32_t *__restrict__ nl, int32_t *__restrict__ sweeps,
                                                                          double *__restrict__ gap_out, int32_t *__restrict__ conv)
{
    __shared__ int32_t s_li[kSlimSolveWarps][kSlimLocal];
    __shared__ double s_w[kSlimSolveWarps][kSlimLocal], s_z[kSlimSolveWarps][kSlimLocal], s_g[kSlimSolveWarps][kSlimLocal];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, r = blockIdx.x * kSlimSolveWarps + wid;
    if (r >= count) return;
    const int j = begin + r, cnt = nl[r];
    const long long base = (long long)r * n;
    const bool local = cnt <= kSlimLocal;
    if (local) {
        for (int s = lane; s < cnt; s += 32) {
            const int k = lidx[base + s];
            s_li[wid][s] = k;
            s_w[wid][s] = w[base + s];
            s_z[wid][s] = z[base + s];
            s_g[wid][s] = diag[k];
        }
        __syncwarp();
    }
    const int32_t *li = local ? s_li[wid] : lidx + base;
    double *wr = local ? s_w[wid] : w + base, *zr = local ? s_z[wid] : z + base;
    const double *qrow = G + (long long)j * n;
    const double yy = diag[j], tol = __dmul_rn(p.tol, yy);
    double gap = slim_gap(qrow, li, wr, zr, cnt, yy, p);
    bool done = gap <= tol;
    int it = 0;
    for (; !done && it < p.max_iter; ++it) {
        double w_max = 0.0, d_w_max = 0.0;
        for (int t = 0; t < cnt; ++t) {
            const int k = li[t];
            const double gkk = local ? s_g[wid][t] : diag[k], wk = wr[t];
            const double tmp = __dadd_rn(zr[t], __dmul_rn(gkk, wk));
            const double nw = tmp > p.l1 ? __ddiv_rn(__dsub_rn(tmp, p.l1), __dadd_rn(gkk, p.l2)) : 0.0;
            const double d = __dsub_rn(nw, wk);
            if (d != 0.0) {          // uniform: every lane read the same wr[t], zr[t]
                __syncwarp();        // ... before lane t % 32 overwrites zr[t] and lane 0 wr[t]
                const double *__restrict__ grow = G + (long long)k * n;
                for (int s = lane; s < cnt; s += 32) zr[s] = __dsub_rn(zr[s], __dmul_rn(d, grow[li[s]]));
                if (lane == 0) wr[t] = nw;
                __syncwarp();
            }
            d_w_max = fmax(d_w_max, fabs(d));
            w_max = fmax(w_max, nw);
        }
        if (w_max == 0.0 || d_w_max / w_max <= p.tol || it == p.max_iter - 1) {
            gap = slim_gap(qrow, li, wr, zr, cnt, yy, p);
            done = gap <= tol;
        }
    }
    if (local) {
        for (int s = lane; s < cnt; s += 32) {
            w[base + s] = s_w[wid][s];
            z[base + s] = s_z[wid][s];
        }
    }
    if (lane == 0) {
        sweeps[r] = it;
        gap_out[r] = gap;
        conv[r] = done;
    }
}

// one CTA per target: the min(nnz - 1, topk) largest coefficients by (value descending, id ascending), by ascending id
__global__ void __launch_bounds__(kSlimThreads) slim_select_kernel(const int32_t *__restrict__ lidx, const double *__restrict__ w,
                                                                   const int32_t *__restrict__ nl, int n, int begin, int topk,
                                                                   int32_t *__restrict__ nbr_idx, float *__restrict__ nbr_val,
                                                                   int32_t *__restrict__ nbr_cnt)
{
    __shared__ int s_warp[kSlimThreads / 32];
    const int r = blockIdx.x, j = begin + r, tid = threadIdx.x, cnt = nl[r];
    const long long base = (long long)r * n;
    // w >= 0, so the fp64 bit pattern orders the values
    auto key = [&](int t) { return (unsigned long long)__double_as_longlong(w[base + t]); };
    int nnz = 0;
    for (int t = tid; t < cnt; t += kSlimThreads) nnz += key(t) != 0ull;
    nnz = slim_block_sum(nnz, s_warp);
    const int keep = nnz - 1 < topk ? nnz - 1 : topk;   // SLiMRecommender.py:89; <= 0 keeps nothing
    // the keep-th largest key: the largest T with #{key >= T} >= keep (bit 63, the sign, is never set)
    unsigned long long T = ~0ull;
    int need = 0;
    if (keep > 0) {
        T = 0ull;
        for (int bit = 62; bit >= 0; --bit) {
            const unsigned long long c = T | (1ull << bit);
            int m = 0;
            for (int t = tid; t < cnt; t += kSlimThreads) m += key(t) >= c;
            if (slim_block_sum(m, s_warp) >= keep) T = c;
        }
        int above = 0;
        for (int t = tid; t < cnt; t += kSlimThreads) above += key(t) > T;
        need = keep - slim_block_sum(above, s_warp);   // ties at T kept, lowest ids first
    }
    int32_t *oi = nbr_idx + (long long)j * topk;
    float *ov = nbr_val + (long long)j * topk;
    int out = 0, ties = 0;
    if (keep > 0) {
        for (int t0 = 0; t0 < cnt; t0 += kSlimThreads) {
            const int t = t0 + tid;
            const unsigned long long k = t < cnt ? key(t) : 0ull;
            int tie_total, sel_total;
            const bool tie = t < cnt && k == T;
            const int tie_rank = slim_flag_rank(tie, s_warp, tie_total);
            const bool sel = t < cnt && (k > T || (tie && ties + tie_rank < need));
            const int pos = slim_flag_rank(sel, s_warp, sel_total);
            if (sel) {
                oi[out + pos] = lidx[base + t];
                ov[out + pos] = __double2float_rn(w[base + t]);
            }
            out += sel_total;
            ties += tie_total;
        }
    }
    for (int t = out + tid; t < topk; t += kSlimThreads) {
        oi[t] = -1;
        ov[t] = 0.f;
    }
    if (tid == 0) nbr_cnt[j] = out;
}

}  // namespace drb

using namespace drb;

extern "C" size_t drb_slim_workspace_bytes(int32_t item_num, int32_t panel)
{
    if (item_num <= 0 || panel <= 0) return 0;
    const size_t n = (size_t)item_num, P = (size_t)panel;
    return 8 * n + P * n * (4 + 8 + 8) + 4 * P;   // diag, then per target: live ids, w, Z; the live counts
}

extern "C" int drb_slim_live(const double *d_G, int32_t item_num, int32_t begin, int32_t count, double l1, int32_t all_live,
                             double *d_diag, int32_t *d_lidx, double *d_w, double *d_z, int32_t *d_nl, void *stream)
{
    DRB_REQUIRE(d_G && d_diag && d_lidx && d_w && d_z && d_nl && item_num > 0 && begin >= 0 && count >= 0 &&
                    (long long)begin + count <= item_num && l1 > 0.0,
                "slim_live: bad arguments (l1 > 0, targets inside [0, item_num))");
    if (count == 0) return DRB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    const double thr = l1 - ldexp(l1, -20);
    slim_diag_kernel<<<grid_for(item_num, 256), 256, 0, st>>>(d_G, item_num, d_diag);
    slim_live_kernel<<<count, kSlimThreads, 0, st>>>(d_G, d_diag, item_num, begin, thr, all_live, d_lidx, d_w, d_z, d_nl);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}

extern "C" int drb_slim_solve(const double *d_G, int32_t item_num, int32_t begin, int32_t count, double l1, double l2, double tol,
                              int32_t max_iter, const double *d_diag, const int32_t *d_lidx, double *d_w, double *d_z,
                              const int32_t *d_nl, int32_t *d_sweeps, double *d_gap, int32_t *d_conv, void *stream)
{
    DRB_REQUIRE(d_G && d_diag && d_lidx && d_w && d_z && d_nl && d_sweeps && d_gap && d_conv && item_num > 0 && begin >= 0 &&
                    count >= 0 && (long long)begin + count <= item_num && l1 > 0.0 && l2 > 0.0 && tol >= 0.0 && max_iter >= 0,
                "slim_solve: bad arguments (l1 > 0, l2 > 0, targets inside [0, item_num))");
    if (count == 0) return DRB_OK;
    const SlimParams p = {l1, l2, tol, max_iter};
    slim_solve_kernel<<<(count + kSlimSolveWarps - 1) / kSlimSolveWarps, kSlimSolveWarps * 32, 0, (cudaStream_t)stream>>>(
        d_G, d_diag, item_num, begin, count, p, d_lidx, d_w, d_z, d_nl, d_sweeps, d_gap, d_conv);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}

extern "C" int drb_slim_select(const int32_t *d_lidx, const double *d_w, const int32_t *d_nl, int32_t item_num, int32_t begin,
                               int32_t count, int32_t topk, int32_t *d_nbr_idx, float *d_nbr_val, int32_t *d_nbr_cnt, void *stream)
{
    DRB_REQUIRE(d_lidx && d_w && d_nl && d_nbr_idx && d_nbr_val && d_nbr_cnt && item_num > 0 && begin >= 0 && count >= 0 &&
                    (long long)begin + count <= item_num && topk >= 1 && topk <= 1024,
                "slim_select: bad arguments (topk in [1, 1024])");
    if (count == 0) return DRB_OK;
    slim_select_kernel<<<count, kSlimThreads, 0, (cudaStream_t)stream>>>(d_lidx, d_w, d_nl, item_num, begin, topk, d_nbr_idx,
                                                                        d_nbr_val, d_nbr_cnt);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}
