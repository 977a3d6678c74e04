// itemknn.cu -- ItemKNNCF (daisy/model/KNNCFRecommender.py, Sarwar et al. 2001 / Ferrari Dacrema et al. 2019) on the device.
//
// The reference's fit is Similarity.compute_similarity: a value transform of X, then for every item column j the products
// g_i = x_i . x_j (fp32), a weight w_i = f(g_i, ss_i, ss_j) in fp32, w_j = 0, and the maxk largest weights with exact zeros
// dropped; W is that sparse [I, I] matrix and pred_mat = X W.  Here g comes from ease.cu's Gram matrix (exact on integer
// data), so what this file adds is:
//
//   drb_itemknn_transform   X' = the transformed fp32 values (the user's mean removed: adjusted; the item's mean removed:
//                           pearson; every stored value 1: jaccard / tanimoto / dice / tversky) and ss_i, the fp32 sum of
//                           x'^2 over item i's stored entries (its square root for the cosine family).  Every sum runs in
//                           fp32 over ascending users / items, the order scipy's products add in.
//   drb_itemknn_neighbours  one CTA per column j reads row j of G (G is symmetric; drb_knn_neighbours_panel takes the rows
//                           j0 .. j0 + rows of G as a panel, which is how UserKNN's [U, U] Gram is consumed) and keeps the min(maxk, I) largest weights
//                           by (weight descending, item id ascending), drops exact zeros and stores the rest by ascending
//                           item id.  Each weight is a few correctly rounded fp32 operations written with the _rn
//                           intrinsics, evaluated left to right as numpy does, so nothing is contracted into an FMA.  The
//                           threshold is found by a 3-pass radix select on the 32-bit ordered key (11 + 11 + 10 bits,
//                           histogram in shared memory); weights are recomputed from the row each pass (it is in L2 after
//                           the first), so no per-column buffer bounds I.
//   drb_itemknn_scores      pred_mat entries: s = sum_{i in N(c)} x_ui W[i, c] in fp64 over ascending i without FMA, the
//                           order and rounding of scipy's csc product; a warp per (user, candidate), each neighbour looked
//                           up in the user's sorted CSR row.
//   drb_itemknn_topk        top-k of each score row by (score descending, position ascending).
#include "common.cuh"
#include "topk.cuh"

namespace drb {

enum { kKnnPlain = 0, kKnnUserMean = 1, kKnnItemMean = 2, kKnnBoolean = 3 };   // drb_itemknn_transform
enum { kKnnCosine = 0, kKnnTanimoto = 1, kKnnDice = 2, kKnnTversky = 3 };      // drb_itemknn_neighbours

// acc + term of lane 0 + term of lane 1 + ... in that order (every lane returns the same sum)
__device__ __forceinline__ float warp_ordered_add(float acc, float term)
{
#pragma unroll
    for (int l = 0; l < 32; ++l) acc = __fadd_rn(acc, __shfl_sync(0xffffffffu, term, l));
    return acc;
}

__device__ __forceinline__ double warp_ordered_add(double acc, double term)
{
#pragma unroll
    for (int l = 0; l < 32; ++l) acc = __dadd_rn(acc, __shfl_sync(0xffffffffu, term, l));
    return acc;
}

// ---------------------------------------------------------------- value transform
// a warp per user: out = in, 1, or in - mean(in over the user's stored entries)
__global__ void knn_user_transform_kernel(const int64_t *__restrict__ row_ptr, const float *__restrict__ in, int U, int transform,
                                          float *__restrict__ out)
{
    const int lane = threadIdx.x & 31;
    for (long long u = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; u < U; u += ((long long)gridDim.x * blockDim.x) >> 5) {
        const long long b = row_ptr[u], e = row_ptr[u + 1];
        float mean = 0.f;
        if (transform == kKnnUserMean && e > b) {
            float sum = 0.f;
            for (long long k0 = b; k0 < e; k0 += 32) sum = warp_ordered_add(sum, k0 + lane < e ? in[k0 + lane] : 0.f);
            mean = __fdiv_rn(sum, (float)(e - b));
        }
        for (long long k = b + lane; k < e; k += 32) out[k] = transform == kKnnBoolean ? 1.f : __fsub_rn(in[k], mean);
    }
}

// a warp per item over its entries in ascending user order (item_ptr / order: the CSR slots grouped by item): removes the
// item's mean when asked, then ss = sum x^2 (or its root)
__global__ void knn_item_transform_kernel(const int64_t *__restrict__ item_ptr, const int32_t *__restrict__ order, int I,
                                          int item_mean, int root, float *__restrict__ val, float *__restrict__ ss)
{
    const int lane = threadIdx.x & 31;
    for (long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < I; i += ((long long)gridDim.x * blockDim.x) >> 5) {
        const long long b = item_ptr[i], e = item_ptr[i + 1];
        float mean = 0.f;
        if (item_mean && e > b) {
            float sum = 0.f;
            for (long long q0 = b; q0 < e; q0 += 32) sum = warp_ordered_add(sum, q0 + lane < e ? val[order[q0 + lane]] : 0.f);
            mean = __fdiv_rn(sum, (float)(e - b));
        }
        float sq = 0.f;
        for (long long q0 = b; q0 < e; q0 += 32) {
            float x = 0.f;
            if (q0 + lane < e) {
                const int k = order[q0 + lane];
                x = val[k];
                if (item_mean) val[k] = x = __fsub_rn(x, mean);
            }
            sq = warp_ordered_add(sq, __fmul_rn(x, x));
        }
        if (lane == 0) ss[i] = root ? __fsqrt_rn(sq) : sq;
    }
}

// ---------------------------------------------------------------- similarity + neighbour selection
struct KnnSim {
    int family, normalize;
    float shrink;
};

// KNNCFRecommender.py:310-337 for one entry of column j, in numpy's fp32 evaluation order
__device__ __forceinline__ float knn_weight(double gram, bool self, float ssj, float ssi, const KnnSim p)
{
    const float g = self ? 0.f : __double2float_rn(gram);
    const float eps = 1e-6f;
    float d;
    if (p.family == kKnnCosine) {
        if (!p.normalize) return p.shrink != 0.f ? __fdiv_rn(g, p.shrink) : g;
        d = __fadd_rn(__fadd_rn(__fmul_rn(ssj, ssi), p.shrink), eps);
    } else if (p.family == kKnnTanimoto) {
        d = __fadd_rn(__fadd_rn(__fsub_rn(__fadd_rn(ssj, ssi), g), p.shrink), eps);
    } else if (p.family == kKnnDice) {
        d = __fadd_rn(__fadd_rn(__fadd_rn(ssj, ssi), p.shrink), eps);
    } else {   // tversky with alpha = beta = 1
        d = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(g, __fsub_rn(ssj, g)), __fsub_rn(ssi, g)), p.shrink), eps);
    }
    return __fmul_rn(g, __fdiv_rn(1.f, d));
}

// 32-bit key ordered as the fp32 weight (-0 counted as +0)
constexpr unsigned kZeroKey = 0x80000000u;
__device__ __forceinline__ unsigned weight_key(float w)
{
    if (w == 0.f) return kZeroKey;
    const unsigned b = __float_as_uint(w);
    return (b >> 31) ? ~b : (b | 0x80000000u);
}

constexpr int kSelThreads = 512;
constexpr int kSelBins = 2048;

// position of this thread's flag among the CTA's set flags (thread order), and their number
__device__ __forceinline__ int block_flag_rank(bool flag, int *s_warp, int &total)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned bal = __ballot_sync(0xffffffffu, flag);
    if (lane == 0) s_warp[warp] = __popc(bal);
    __syncthreads();
    int before = 0, all = 0;
#pragma unroll
    for (int w = 0; w < kSelThreads / 32; ++w) {
        const int c = s_warp[w];
        before += w < warp ? c : 0;
        all += c;
    }
    __syncthreads();
    total = all;
    return before + __popc(bal & ((1u << lane) - 1u));
}

// one CTA per row of a panel of G: row r holds column j = j0 + r (G is symmetric), ld entries apart
__global__ void __launch_bounds__(kSelThreads) knn_select_kernel(const double *__restrict__ G, long long ld, int j0, int n,
                                                                 const float *__restrict__ ss, const KnnSim p, int keep, int maxk,
                                                                 int32_t *__restrict__ nbr_idx, float *__restrict__ nbr_val,
                                                                 int32_t *__restrict__ nbr_cnt)
{
    __shared__ unsigned hist[kSelBins];
    __shared__ int s_warp[kSelThreads / 32];
    __shared__ unsigned s_prefix;
    __shared__ int s_need;
    const int j = j0 + blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const double *row = G + (long long)blockIdx.x * ld;
    const float ssj = ss[j];

    // radix select: after the three passes `prefix` is the key of the keep-th largest weight and `need` how many weights
    // with exactly that key belong to the top
    unsigned prefix = 0, mask = 0;
    int need = keep;
    for (int pass = 0; pass < 3; ++pass) {
        const int shift = pass == 0 ? 21 : pass == 1 ? 10 : 0, bins = pass == 2 ? 1024 : 2048;
        for (int t = tid; t < kSelBins; t += kSelThreads) hist[t] = 0;
        __syncthreads();
        unsigned zeros = 0;   // most weights of a sparse column are 0: counted in registers, not on one shared counter
        for (int i = tid; i < n; i += kSelThreads) {
            const unsigned key = weight_key(knn_weight(row[i], i == j, ssj, ss[i], p));
            if ((key & mask) != prefix) continue;
            if (key == kZeroKey) ++zeros; else atomicAdd(&hist[(key >> shift) & (bins - 1)], 1u);
        }
        zeros = __reduce_add_sync(0xffffffffu, zeros);
        if (lane == 0 && zeros) atomicAdd(&hist[(kZeroKey >> shift) & (bins - 1)], zeros);
        __syncthreads();
        if (warp == 0) {   // lane l owns the l-th group of bins from the top
            const int per = bins / 32, top = bins - lane * per;
            unsigned mine = 0;
            for (int b = top - per; b < top; ++b) mine += hist[b];
            unsigned inc = mine;
#pragma unroll
            for (int off = 1; off < 32; off <<= 1) {
                const unsigned t = __shfl_up_sync(0xffffffffu, inc, off);
                if (lane >= off) inc += t;
            }
            unsigned above = inc - mine;
            if (above < (unsigned)need && (unsigned)need <= inc) {
                int b = top - 1;
                while (above + hist[b] < (unsigned)need) above += hist[b--];
                s_prefix = prefix | ((unsigned)b << shift);
                s_need = need - (int)above;
            }
        }
        __syncthreads();
        prefix = s_prefix;
        need = s_need;
        mask |= (unsigned)(bins - 1) << shift;
    }

    // collect in item order: keys above the threshold, then the first `need` ties by item id; exact zeros are not stored
    int32_t *oi = nbr_idx + (long long)j * maxk;
    float *ov = nbr_val + (long long)j * maxk;
    int count = 0, ties = 0;
    for (int i0 = 0; i0 < n; i0 += kSelThreads) {
        const int i = i0 + tid;
        float w = 0.f;
        unsigned key = 0;
        if (i < n) {
            w = knn_weight(row[i], i == j, ssj, ss[i], p);
            key = weight_key(w);
        }
        int tie_total = 0, sel_total;
        const bool tie = i < n && key == prefix;
        int tie_rank = 0;
        if (prefix != kZeroKey) tie_rank = block_flag_rank(tie, s_warp, tie_total);   // uniform branch; zero ties are dropped anyway
        const bool sel = i < n && key != kZeroKey && (key > prefix || (tie && ties + tie_rank < need));
        const int pos = block_flag_rank(sel, s_warp, sel_total);
        if (sel) {
            oi[count + pos] = i;
            ov[count + pos] = w;
        }
        count += sel_total;
        ties += tie_total;
    }
    for (int t = count + tid; t < maxk; t += kSelThreads) {
        oi[t] = -1;
        ov[t] = 0.f;
    }
    if (tid == 0) nbr_cnt[j] = count;
}

// ---------------------------------------------------------------- scoring
constexpr int kScoreWarps = 8;

// grid (rows, ceil(C / kScoreWarps)): a warp per candidate c of row's user
__global__ void __launch_bounds__(kScoreWarps * 32) knn_scores_kernel(const int64_t *__restrict__ row_ptr, const int32_t *__restrict__ col,
                                                                      const float *__restrict__ val, const int32_t *__restrict__ nbr_idx,
                                                                      const float *__restrict__ nbr_val, const int32_t *__restrict__ nbr_cnt,
                                                                      int maxk, const int64_t *__restrict__ users,
                                                                      const int64_t *__restrict__ cands, int C, double *__restrict__ scores)
{
    const int lane = threadIdx.x & 31, c = blockIdx.y * kScoreWarps + (threadIdx.x >> 5);
    if (c >= C) return;
    const long long r = blockIdx.x, u = users[r], b = row_ptr[u], e = row_ptr[u + 1];
    const long long item = cands ? cands[r * C + c] : c;
    const int cnt = e > b ? nbr_cnt[item] : 0;
    double acc = 0.0;
    for (int q0 = 0; q0 < cnt; q0 += 32) {
        double term = 0.0;
        if (q0 + lane < cnt) {
            const int i = nbr_idx[item * maxk + q0 + lane];
            long long lo = b, hi = e - 1;
            while (lo < hi) {
                const long long mid = (lo + hi) >> 1;
                if (col[mid] < i) lo = mid + 1; else hi = mid;
            }
            if (col[lo] == i) term = __dmul_rn((double)val[lo], (double)nbr_val[item * maxk + q0 + lane]);
        }
        acc = warp_ordered_add(acc, term);
    }
    if (lane == 0) scores[r * C + c] = acc;
}

template <int kThreads>
__global__ void __launch_bounds__(kThreads) knn_topk_kernel(const double *__restrict__ scores, int C, int k,
                                                            const int64_t *__restrict__ cands, int64_t *__restrict__ out)
{
    const long long r = blockIdx.x;
    block_topk(scores + r * C, C, k, cands ? cands + r * C : nullptr, out + r * k);
}

}  // namespace drb

using namespace drb;

extern "C" int drb_itemknn_transform(const int64_t *d_row_ptr, const float *d_val_in, int32_t user_num, int32_t item_num,
                                     const int64_t *d_item_ptr, const int32_t *d_item_order, int32_t transform, int32_t root,
                                     float *d_val_out, float *d_ss, void *stream)
{
    DRB_REQUIRE(d_row_ptr && d_item_ptr && d_val_out && d_ss && user_num > 0 && item_num > 0 && transform >= kKnnPlain &&
                    transform <= kKnnBoolean,
                "itemknn_transform: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    knn_user_transform_kernel<<<grid_for((long long)user_num * 32, 256), 256, 0, st>>>(d_row_ptr, d_val_in, user_num, transform,
                                                                                      d_val_out);
    knn_item_transform_kernel<<<grid_for((long long)item_num * 32, 256), 256, 0, st>>>(d_item_ptr, d_item_order, item_num,
                                                                                      transform == kKnnItemMean, root, d_val_out, d_ss);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}

extern "C" int drb_knn_neighbours_panel(const double *d_G, int32_t n, int32_t j0, int32_t rows, const float *d_ss, int32_t family,
                                        int32_t normalize, float shrink, int32_t maxk, int32_t *d_nbr_idx, float *d_nbr_val,
                                        int32_t *d_nbr_cnt, void *stream)
{
    DRB_REQUIRE(d_G && d_ss && d_nbr_idx && d_nbr_val && d_nbr_cnt && n > 0 && j0 >= 0 && rows >= 0 && j0 + rows <= n &&
                    family >= kKnnCosine && family <= kKnnTversky && maxk >= 1 && maxk <= 1024,
                "itemknn_neighbours: bad arguments (maxk in [1, 1024])");
    if (rows == 0) return DRB_OK;
    const KnnSim p = {family, family == kKnnCosine ? normalize : 0, shrink};
    knn_select_kernel<<<rows, kSelThreads, 0, (cudaStream_t)stream>>>(d_G, n, j0, n, d_ss, p, maxk < n ? maxk : n, maxk, d_nbr_idx,
                                                                      d_nbr_val, d_nbr_cnt);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}

extern "C" int drb_itemknn_neighbours(const double *d_G, int32_t n, const float *d_ss, int32_t family, int32_t normalize,
                                      float shrink, int32_t maxk, int32_t *d_nbr_idx, float *d_nbr_val, int32_t *d_nbr_cnt,
                                      void *stream)
{
    return drb_knn_neighbours_panel(d_G, n, 0, n, d_ss, family, normalize, shrink, maxk, d_nbr_idx, d_nbr_val, d_nbr_cnt, stream);
}

extern "C" int drb_itemknn_scores(const int64_t *d_row_ptr, const int32_t *d_col, const float *d_val, const int32_t *d_nbr_idx,
                                  const float *d_nbr_val, const int32_t *d_nbr_cnt, int32_t maxk, int32_t item_num,
                                  const int64_t *d_users, int64_t n_rows, const int64_t *d_cands, int32_t cand_num, double *d_scores,
                                  void *stream)
{
    DRB_REQUIRE(d_row_ptr && d_nbr_idx && d_nbr_val && d_nbr_cnt && d_users && d_scores && maxk > 0 && item_num > 0 && n_rows >= 0 &&
                    n_rows < (1ll << 31) && cand_num > 0 && (d_cands || cand_num == item_num) &&
                    (cand_num + kScoreWarps - 1) / kScoreWarps <= 65535,
                "itemknn_scores: bad arguments");
    if (n_rows == 0) return DRB_OK;
    knn_scores_kernel<<<dim3((unsigned)n_rows, (cand_num + kScoreWarps - 1) / kScoreWarps), kScoreWarps * 32, 0, (cudaStream_t)stream>>>(
        d_row_ptr, d_col, d_val, d_nbr_idx, d_nbr_val, d_nbr_cnt, maxk, d_users, d_cands, cand_num, d_scores);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}

extern "C" int drb_itemknn_topk(const double *d_scores, int64_t n_rows, int32_t cand_num, const int64_t *d_cands, int32_t topk,
                                int64_t *d_out, void *stream)
{
    DRB_REQUIRE(d_scores && d_out && n_rows >= 0 && n_rows < (1ll << 31) && cand_num > 0 && topk > 0 && topk <= cand_num,
                "itemknn_topk: bad arguments");
    if (n_rows == 0) return DRB_OK;
    if (cand_num > 4096)
        knn_topk_kernel<1024><<<(unsigned)n_rows, 1024, 0, (cudaStream_t)stream>>>(d_scores, cand_num, topk, d_cands, d_out);
    else
        knn_topk_kernel<256><<<(unsigned)n_rows, 256, 0, (cudaStream_t)stream>>>(d_scores, cand_num, topk, d_cands, d_out);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}
