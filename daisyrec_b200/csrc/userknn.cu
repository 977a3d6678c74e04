// userknn.cu -- UserKNNCF (daisy/model/KNNCFRecommender.py:459-536) on the device.
//
// The reference runs ItemKNN's Similarity on X^T [I, U]: its columns are users, so W is [U, U] with column j holding the
// neighbours of user j, and then pred_mat = W X (:510) -- W multiplies from the LEFT.  pred[u, c] = sum_v W[u, v] x_vc, and
// W[u, v] != 0 exactly when u is one of v's neighbours: a user's score sums over its REVERSE neighbours.  The similarity
// itself runs on itemknn.cu's transform and selection and ease.cu's panelled Gram; what this file adds is:
//
//   drb_userknn_transpose  X^T's values and the slot map of X into X^T: for each slot k of X (user u, item i) its position in
//                          X^T's row i (the drb_csr_build CSR of the (item, user) pairs), t_val[pos] = val[k], order[k] = pos.
//                          X's row pointer and `order` are then X^T's slots grouped by user in ascending item order, the
//                          grouping drb_itemknn_transform reads.
//   drb_userknn_reverse    the forward lists (KnnNeighbours: N(v) by ascending id) turned into R(u) = {v : u in N(v)} as a CSR
//                          over u with ascending v: the (u, v) pairs go through drb_csr_build (no bound on a row's length),
//                          then each value W[u, v] is placed by a binary search for v in row u.
//   drb_userknn_scores     pred_mat entries for (user, candidate) pairs: s = sum_{v in R(u)} W[u, v] x_vc in fp64 over ascending
//                          v without FMA -- the order of scipy's csc product, which runs csr_matmat on the transposes and adds,
//                          for each (c, u), the terms of the users v of item c in ascending v.  A warp per (user, candidate),
//                          each x_vc looked up in v's sorted CSR row.
//   drb_userknn_full_scores  the same sums over every item: one CTA per user walks R(u) in order and scatters each row of X
//                          into the user's fp64 score row; a barrier between rows keeps every entry's additions in v order.
#include "common.cuh"

namespace drb {

// a warp per user: each of the user's X slots finds its position in X^T's row of its item
__global__ void userknn_transpose_kernel(const int64_t *__restrict__ row_ptr, const int32_t *__restrict__ col,
                                         const float *__restrict__ val, int U, const int64_t *__restrict__ t_ptr,
                                         const int32_t *__restrict__ t_col, float *__restrict__ t_val, int32_t *__restrict__ order)
{
    const int lane = threadIdx.x & 31;
    for (long long u = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; u < U; u += ((long long)gridDim.x * blockDim.x) >> 5) {
        for (long long k = row_ptr[u] + lane; k < row_ptr[u + 1]; k += 32) {
            const int i = col[k];
            long long lo = t_ptr[i], hi = t_ptr[i + 1] - 1;   // u is in the row: both CSRs hold the same pairs
            while (lo < hi) {
                const long long mid = (lo + hi) >> 1;
                if (t_col[mid] < u) lo = mid + 1; else hi = mid;
            }
            t_val[lo] = val[k];
            order[k] = (int32_t)lo;
        }
    }
}

// one (u, v) pair per slot of the forward lists; an empty slot goes to the extra row n (dropped after the build)
__global__ void userknn_pairs_kernel(const int32_t *__restrict__ nbr_idx, const int32_t *__restrict__ nbr_cnt, int n, int maxk,
                                     int32_t *__restrict__ pu, int32_t *__restrict__ pv)
{
    const long long total = (long long)n * maxk;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < total; k += (long long)gridDim.x * blockDim.x) {
        const int v = (int)(k / maxk), q = (int)(k % maxk);
        const bool live = q < nbr_cnt[v];
        pu[k] = live ? nbr_idx[k] : n;
        pv[k] = live ? v : 0;
    }
}

// r_val[slot of (u, v)] = W[u, v]: each forward entry finds v in row u of R
__global__ void userknn_place_kernel(const int32_t *__restrict__ nbr_idx, const float *__restrict__ nbr_val,
                                     const int32_t *__restrict__ nbr_cnt, int n, int maxk, const int64_t *__restrict__ r_ptr,
                                     const int32_t *__restrict__ r_col, float *__restrict__ r_val)
{
    const long long total = (long long)n * maxk;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < total; k += (long long)gridDim.x * blockDim.x) {
        const int v = (int)(k / maxk), q = (int)(k % maxk);
        if (q >= nbr_cnt[v]) continue;
        const int u = nbr_idx[k];
        long long lo = r_ptr[u], hi = r_ptr[u + 1] - 1;
        while (lo < hi) {
            const long long mid = (lo + hi) >> 1;
            if (r_col[mid] < v) lo = mid + 1; else hi = mid;
        }
        r_val[lo] = nbr_val[k];
    }
}

// acc + term of lane 0 + term of lane 1 + ... in that order (every lane returns the same sum)
__device__ __forceinline__ double warp_ordered_add(double acc, double term)
{
#pragma unroll
    for (int l = 0; l < 32; ++l) acc = __dadd_rn(acc, __shfl_sync(0xffffffffu, term, l));
    return acc;
}

constexpr int kScoreWarps = 8;

// grid (rows, ceil(C / kScoreWarps)): a warp per candidate c of the row's user
__global__ void __launch_bounds__(kScoreWarps * 32) userknn_scores_kernel(const int64_t *__restrict__ row_ptr, const int32_t *__restrict__ col,
                                                                          const float *__restrict__ val, const int64_t *__restrict__ r_ptr,
                                                                          const int32_t *__restrict__ r_col, const float *__restrict__ r_val,
                                                                          const int64_t *__restrict__ users, const int64_t *__restrict__ cands,
                                                                          int C, double *__restrict__ scores)
{
    const int lane = threadIdx.x & 31, c = blockIdx.y * kScoreWarps + (threadIdx.x >> 5);
    if (c >= C) return;
    const long long r = blockIdx.x, u = users[r], b = r_ptr[u], e = r_ptr[u + 1];
    const int item = (int)cands[r * C + c];
    double acc = 0.0;
    for (long long q0 = b; q0 < e; q0 += 32) {
        double term = 0.0;
        if (q0 + lane < e) {
            const int v = r_col[q0 + lane];
            long long lo = row_ptr[v], hi = row_ptr[v + 1] - 1;
            if (hi >= lo) {
                while (lo < hi) {
                    const long long mid = (lo + hi) >> 1;
                    if (col[mid] < item) lo = mid + 1; else hi = mid;
                }
                if (col[lo] == item) term = __dmul_rn((double)val[lo], (double)r_val[q0 + lane]);
            }
        }
        acc = warp_ordered_add(acc, term);
    }
    if (lane == 0) scores[r * C + c] = acc;
}

constexpr int kFullThreads = 256;

// one CTA per row: scores[row][:] = sum over v in R(u), ascending, of W[u, v] x_v (an item appears once per row of X, so
// the threads of one v never meet; the barrier orders the v)
__global__ void __launch_bounds__(kFullThreads) userknn_full_scores_kernel(const int64_t *__restrict__ row_ptr, const int32_t *__restrict__ col,
                                                                           const float *__restrict__ val, const int64_t *__restrict__ r_ptr,
                                                                           const int32_t *__restrict__ r_col, const float *__restrict__ r_val,
                                                                           int I, const int64_t *__restrict__ users, double *__restrict__ scores)
{
    const long long r = blockIdx.x, u = users[r];
    double *sc = scores + r * I;
    for (int c = threadIdx.x; c < I; c += kFullThreads) sc[c] = 0.0;
    __syncthreads();
    for (long long q = r_ptr[u]; q < r_ptr[u + 1]; ++q) {
        const int v = r_col[q];
        const double w = (double)r_val[q];
        for (long long k = row_ptr[v] + threadIdx.x; k < row_ptr[v + 1]; k += kFullThreads)
            sc[col[k]] = __dadd_rn(sc[col[k]], __dmul_rn((double)val[k], w));
        __syncthreads();
    }
}

}  // namespace drb

using namespace drb;

extern "C" int drb_userknn_transpose(const int64_t *d_row_ptr, const int32_t *d_col, const float *d_val, int32_t user_num,
                                     const int64_t *d_t_ptr, const int32_t *d_t_col, float *d_t_val, int32_t *d_order, void *stream)
{
    DRB_REQUIRE(d_row_ptr && d_t_ptr && user_num > 0, "userknn_transpose: bad arguments");
    userknn_transpose_kernel<<<grid_for((long long)user_num * 32, 256), 256, 0, (cudaStream_t)stream>>>(
        d_row_ptr, d_col, d_val, user_num, d_t_ptr, d_t_col, d_t_val, d_order);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}

extern "C" int drb_userknn_pairs(const int32_t *d_nbr_idx, const int32_t *d_nbr_cnt, int32_t n, int32_t maxk, int32_t *d_pu,
                                 int32_t *d_pv, void *stream)
{
    DRB_REQUIRE(d_nbr_idx && d_nbr_cnt && d_pu && d_pv && n > 0 && maxk > 0, "userknn_pairs: bad arguments");
    userknn_pairs_kernel<<<grid_for((long long)n * maxk, 256), 256, 0, (cudaStream_t)stream>>>(d_nbr_idx, d_nbr_cnt, n, maxk, d_pu,
                                                                                               d_pv);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}

extern "C" int drb_userknn_place(const int32_t *d_nbr_idx, const float *d_nbr_val, const int32_t *d_nbr_cnt, int32_t n, int32_t maxk,
                                 const int64_t *d_r_ptr, const int32_t *d_r_col, float *d_r_val, void *stream)
{
    DRB_REQUIRE(d_nbr_idx && d_nbr_val && d_nbr_cnt && d_r_ptr && n > 0 && maxk > 0, "userknn_place: bad arguments");
    userknn_place_kernel<<<grid_for((long long)n * maxk, 256), 256, 0, (cudaStream_t)stream>>>(d_nbr_idx, d_nbr_val, d_nbr_cnt, n, maxk,
                                                                                               d_r_ptr, d_r_col, d_r_val);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}

extern "C" int drb_userknn_scores(const int64_t *d_row_ptr, const int32_t *d_col, const float *d_val, const int64_t *d_r_ptr,
                                  const int32_t *d_r_col, const float *d_r_val, const int64_t *d_users, int64_t n_rows,
                                  const int64_t *d_cands, int32_t cand_num, double *d_scores, void *stream)
{
    DRB_REQUIRE(d_row_ptr && d_r_ptr && d_users && d_cands && d_scores && n_rows >= 0 && n_rows < (1ll << 31) && cand_num > 0 &&
                    (cand_num + kScoreWarps - 1) / kScoreWarps <= 65535,
                "userknn_scores: bad arguments");
    if (n_rows == 0) return DRB_OK;
    userknn_scores_kernel<<<dim3((unsigned)n_rows, (cand_num + kScoreWarps - 1) / kScoreWarps), kScoreWarps * 32, 0,
                            (cudaStream_t)stream>>>(d_row_ptr, d_col, d_val, d_r_ptr, d_r_col, d_r_val, d_users, d_cands, cand_num,
                                                    d_scores);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}

extern "C" int drb_userknn_full_scores(const int64_t *d_row_ptr, const int32_t *d_col, const float *d_val, const int64_t *d_r_ptr,
                                       const int32_t *d_r_col, const float *d_r_val, int32_t item_num, const int64_t *d_users,
                                       int64_t n_rows, double *d_scores, void *stream)
{
    DRB_REQUIRE(d_row_ptr && d_r_ptr && d_users && d_scores && item_num > 0 && n_rows >= 0 && n_rows < (1ll << 31),
                "userknn_full_scores: bad arguments");
    if (n_rows == 0) return DRB_OK;
    userknn_full_scores_kernel<<<(unsigned)n_rows, kFullThreads, 0, (cudaStream_t)stream>>>(d_row_ptr, d_col, d_val, d_r_ptr, d_r_col,
                                                                                           d_r_val, item_num, d_users, d_scores);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}
