// rank.cu -- fused gather + GEMV + top-K selection for MF.rank / MF.full_rank / MF.predict.
//
// Stands behind daisy/model/MFRecommender.py:99-133.  The reference materialises
// Q[cands] as a [128, 1000, F] tensor, runs bmm, a FULL argsort of every row, a gather and a
// slice (:113-119); full_rank does matmul + full argsort over all items (:131-133).  Here one CTA
// owns one user: its factor row sits in registers, lane groups stream candidate / item rows with
// 128-bit loads, reduce the dot product in the canonical order (so scores are reproducible bit for
// bit, see oracle orc_dot) and write 64-bit sort keys (~ordered(score) << 32 | position) to shared
// memory; a block-wide bitonic network orders them and the first K ids are written out.
// Candidate lists longer than the key buffer are consumed in chunks that are merged with the
// running best K (the full_rank path for item_num > 4096).
// Ties (equal fp32 score): lower candidate position / lower item id first.
#include "common.cuh"

namespace drb {

constexpr int kRankThreads = 256;
constexpr int kRankMaxKeys = 4096;

__device__ __forceinline__ unsigned long long make_key(float score, unsigned pos)
{
    score += 0.0f;                                   // -0.0 -> +0.0: equal scores must compare equal
    unsigned u = __float_as_uint(score);
    u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);  // monotone map float -> unsigned (ascending)
    return ((unsigned long long)(~u) << 32) | pos;   // ascending key order == descending score, then position
}

__device__ __forceinline__ void bitonic_sort(unsigned long long *a, int n, int tid)
{
    for (int k = 2; k <= n; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = tid; i < n; i += kRankThreads) {
                int ixj = i ^ j;
                if (ixj > i) {
                    unsigned long long x = a[i], y = a[ixj];
                    bool asc = (i & k) == 0;
                    if ((x > y) == asc) {
                        a[i] = y;
                        a[ixj] = x;
                    }
                }
            }
            __syncthreads();
        }
    }
}

// MODE 0: candidate lists (ids from cands[row, :], output float32 ids)   -- MF.rank
// MODE 1: all items 0..count-1 (output int64 ids)                          -- MF.full_rank
template <int VEC, int W, int NCH, int MODE>
__global__ void __launch_bounds__(kRankThreads) rank_kernel(const float *__restrict__ P, const float *__restrict__ Q, int F,
                                                            const int64_t *__restrict__ users,
                                                            const int64_t *__restrict__ cands, int count, int K, int nkeys,
                                                            float *__restrict__ out_f, int64_t *__restrict__ out_i,
                                                            const float *__restrict__ bias, int U, int I)
{
    extern __shared__ unsigned long long keys[];
    constexpr int GPW = 32 / W, GROUPS = (kRankThreads / 32) * GPW;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int gl = lane % W, group = warp * GPW + lane / W;
    const int chunks = F / VEC;
    const long long row = blockIdx.x;
    const Row<VEC, W, NCH> p = load_row<VEC, W, NCH>(P + (size_t)users[row] * F, gl, chunks, true);
    const int64_t *crow = (MODE == 0) ? cands + row * count : nullptr;

    int done = 0;
    bool first = true;
    while (done < count) {
        const int lo = first ? 0 : K;                 // keys[0..K) keep the running best after the first chunk
        const int take = min(count - done, nkeys - lo);
        for (int i = tid + lo + take; i < nkeys; i += kRankThreads) keys[i] = ~0ull;  // sentinels sort last
        for (int c0 = 0; c0 < take; c0 += GROUPS) {
            int c = c0 + group;
            bool ok = c < take;
            long long item = 0;
            if (ok) item = (MODE == 0) ? crow[done + c] : (long long)(done + c);
            Row<VEC, W, NCH> q = load_row<VEC, W, NCH>(Q + (size_t)item * F, gl, chunks, ok);
            float s = dot_rows<VEC, W, NCH>(p, q);
            // FM (FMRecommender.py:113,129): scores += (u_bias(u) + i_bias(c)) + bias_
            if (bias != nullptr) s += (bias[users[row]] + bias[U + item]) + bias[U + I];
            if (ok && gl == 0) keys[lo + c] = make_key(s, (unsigned)(done + c));
        }
        __syncthreads();
        bitonic_sort(keys, nkeys, tid);
        done += take;
        first = false;
    }
    for (int k = tid; k < K; k += kRankThreads) {
        unsigned pos = (unsigned)(keys[k] & 0xffffffffull);
        if (MODE == 0)
            out_f[row * K + k] = (float)crow[pos];
        else
            out_i[row * K + k] = (int64_t)pos;
    }
}

// top-K of PRE-COMPUTED scores (NeuMF: the scores come out of the tower).  MODE as in rank_kernel.
template <int MODE>
__global__ void __launch_bounds__(kRankThreads) topk_scores_kernel(const float *__restrict__ scores,
                                                                   const int64_t *__restrict__ cands, int count, int K,
                                                                   int nkeys, float *__restrict__ out_f,
                                                                   int64_t *__restrict__ out_i)
{
    extern __shared__ unsigned long long keys[];
    const int tid = threadIdx.x;
    const long long row = blockIdx.x;
    const float *srow = scores + row * count;
    const int64_t *crow = (MODE == 0) ? cands + row * count : nullptr;
    int done = 0;
    bool first = true;
    while (done < count) {
        const int lo = first ? 0 : K;
        const int take = min(count - done, nkeys - lo);
        for (int i = tid + lo + take; i < nkeys; i += kRankThreads) keys[i] = ~0ull;
        for (int c = tid; c < take; c += kRankThreads) keys[lo + c] = make_key(srow[done + c], (unsigned)(done + c));
        __syncthreads();
        bitonic_sort(keys, nkeys, tid);
        done += take;
        first = false;
    }
    for (int k = tid; k < K; k += kRankThreads) {
        unsigned pos = (unsigned)(keys[k] & 0xffffffffull);
        if (MODE == 0)
            out_f[row * K + k] = (float)crow[pos];
        else
            out_i[row * K + k] = (int64_t)pos;
    }
}

template <int VEC, int W, int NCH>
__global__ void predict_kernel(const float *__restrict__ P, const float *__restrict__ Q, int F, const int32_t *__restrict__ u,
                               const int32_t *__restrict__ it, long long n, float *__restrict__ out,
                               const float *__restrict__ bias, int U, int I)
{
    constexpr int GPW = 32 / W;
    const int lane = threadIdx.x & 31, gl = lane % W;
    const int chunks = F / VEC;
    long long groups_total = (long long)gridDim.x * (blockDim.x / 32) * GPW;
    long long g0 = ((long long)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5)) * GPW + lane / W;
    long long rounds = (n + groups_total - 1) / groups_total;
    for (long long r = 0; r < rounds; ++r) {
        long long t = r * groups_total + g0;
        bool ok = t < n;
        int uu = ok ? u[t] : 0, ii = ok ? it[t] : 0;
        Row<VEC, W, NCH> a = load_row<VEC, W, NCH>(P + (size_t)uu * F, gl, chunks, ok);
        Row<VEC, W, NCH> b = load_row<VEC, W, NCH>(Q + (size_t)ii * F, gl, chunks, ok);
        float s = dot_rows<VEC, W, NCH>(a, b);
        if (bias != nullptr) s += (bias[uu] + bias[U + ii]) + bias[U + I];     // FM.forward (FMRecommender.py:66-67)
        if (ok && gl == 0) out[t] = s;
    }
}

typedef void (*RankKernel)(const float *, const float *, int, const int64_t *, const int64_t *, int, int, int, float *,
                           int64_t *, const float *, int, int);
typedef void (*PredictKernel)(const float *, const float *, int, const int32_t *, const int32_t *, long long, float *,
                              const float *, int, int);

template <int VEC, int MODE>
static RankKernel pick_rank_v(int W, int NCH)
{
#define DRB_CASE(w, n) \
    if (W == w && NCH == n) return rank_kernel<VEC, w, n, MODE>;
    DRB_CASE(1, 1) DRB_CASE(2, 1) DRB_CASE(4, 1) DRB_CASE(8, 1) DRB_CASE(16, 1) DRB_CASE(32, 1)
    DRB_CASE(32, 2) DRB_CASE(32, 4) DRB_CASE(32, 8)
#undef DRB_CASE
    return nullptr;
}
template <int MODE>
static RankKernel pick_rank(int F)
{
    RowGeom g = row_geom(F);
    if (g.vec == 4) return pick_rank_v<4, MODE>(g.width, g.nch);
    if (g.vec == 2) return pick_rank_v<2, MODE>(g.width, g.nch);
    return pick_rank_v<1, MODE>(g.width, g.nch);
}
template <int VEC>
static PredictKernel pick_predict_v(int W, int NCH)
{
#define DRB_CASE(w, n) \
    if (W == w && NCH == n) return predict_kernel<VEC, w, n>;
    DRB_CASE(1, 1) DRB_CASE(2, 1) DRB_CASE(4, 1) DRB_CASE(8, 1) DRB_CASE(16, 1) DRB_CASE(32, 1)
    DRB_CASE(32, 2) DRB_CASE(32, 4) DRB_CASE(32, 8)
#undef DRB_CASE
    return nullptr;
}

static int launch_rank(int mode, const float *P, const float *Q, int F, const int64_t *users, long long n,
                       const int64_t *cands, int count, int K, float *out_f, int64_t *out_i, cudaStream_t st,
                       const float *bias = nullptr, int U = 0, int I = 0)
{
    DRB_REQUIRE(P && Q && users && F > 0 && count > 0 && K > 0 && n >= 0, "rank: bad arguments");
    DRB_REQUIRE(K <= count, "rank: topk=%d exceeds the %d scored ids", K, count);
    DRB_REQUIRE(2 * K <= kRankMaxKeys, "rank: topk=%d too large (max %d)", K, kRankMaxKeys / 2);
    if (n == 0) return DRB_OK;
    RankKernel k = mode == 0 ? pick_rank<0>(F) : pick_rank<1>(F);
    DRB_REQUIRE(k != nullptr, "unsupported factors=%d", F);
    int nkeys = 64;
    while (nkeys < count && nkeys < kRankMaxKeys) nkeys <<= 1;
    while (nkeys < 2 * K) nkeys <<= 1;
    size_t smem = sizeof(unsigned long long) * (size_t)nkeys;
    DRB_REQUIRE(n <= 0x7fffffffLL, "rank: too many users in one call");
    k<<<(unsigned)n, kRankThreads, smem, st>>>(P, Q, F, users, cands, count, K, nkeys, out_f, out_i, bias, U, I);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}

}  // namespace drb

using namespace drb;

extern "C" int drb_mf_rank(const float *d_P, const float *d_Q, int32_t F, const int64_t *d_users, int64_t n_users,
                           const int64_t *d_cands, int32_t cand_num, int32_t topk, float *d_out, void *stream)
{
    DRB_REQUIRE(d_cands && d_out, "mf_rank: null argument");
    return launch_rank(0, d_P, d_Q, F, d_users, n_users, d_cands, cand_num, topk, d_out, nullptr, (cudaStream_t)stream);
}

extern "C" int drb_mf_full_rank(const float *d_P, const float *d_Q, int32_t F, int32_t item_num, const int64_t *d_users,
                                int64_t n_users, int32_t topk, int64_t *d_out, void *stream)
{
    DRB_REQUIRE(d_out, "mf_full_rank: null argument");
    return launch_rank(1, d_P, d_Q, F, d_users, n_users, nullptr, item_num, topk, nullptr, d_out, (cudaStream_t)stream);
}

extern "C" int drb_topk_from_scores(const float *d_scores, const int64_t *d_cands, int64_t n_rows, int32_t count, int32_t topk,
                                    float *d_out_f, int64_t *d_out_i, void *stream)
{
    DRB_REQUIRE(d_scores && count > 0 && topk > 0 && topk <= count && n_rows >= 0 && 2 * topk <= kRankMaxKeys &&
                    ((d_cands && d_out_f) || (!d_cands && d_out_i)),
                "topk_from_scores: bad arguments");
    if (n_rows == 0) return DRB_OK;
    int nkeys = 64;
    while (nkeys < count && nkeys < kRankMaxKeys) nkeys <<= 1;
    while (nkeys < 2 * topk) nkeys <<= 1;
    size_t smem = sizeof(unsigned long long) * (size_t)nkeys;
    if (d_cands)
        topk_scores_kernel<0><<<(unsigned)n_rows, kRankThreads, smem, (cudaStream_t)stream>>>(d_scores, d_cands, count, topk, nkeys,
                                                                                             d_out_f, nullptr);
    else
        topk_scores_kernel<1><<<(unsigned)n_rows, kRankThreads, smem, (cudaStream_t)stream>>>(d_scores, nullptr, count, topk,
                                                                                             nkeys, nullptr, d_out_i);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}

static int launch_predict(const float *d_P, const float *d_Q, int32_t F, const int32_t *d_u, const int32_t *d_i, int64_t n,
                          float *d_out, void *stream, const float *d_bias, int U, int I)
{
    DRB_REQUIRE(d_P && d_Q && d_u && d_i && d_out && F > 0 && n >= 0, "predict: bad arguments");
    if (n == 0) return DRB_OK;
    RowGeom g = row_geom(F);
    PredictKernel k = g.vec == 4 ? pick_predict_v<4>(g.width, g.nch)
                                 : g.vec == 2 ? pick_predict_v<2>(g.width, g.nch) : pick_predict_v<1>(g.width, g.nch);
    DRB_REQUIRE(k != nullptr, "unsupported factors=%d", F);
    const int per_block = (256 / 32) * (32 / g.width);
    k<<<grid_for(n, per_block, 8), 256, 0, (cudaStream_t)stream>>>(d_P, d_Q, F, d_u, d_i, n, d_out, d_bias, U, I);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}

extern "C" int drb_mf_predict(const float *d_P, const float *d_Q, int32_t F, const int32_t *d_u, const int32_t *d_i,
                              int64_t n, float *d_out, void *stream)
{
    return launch_predict(d_P, d_Q, F, d_u, d_i, n, d_out, stream, nullptr, 0, 0);
}

// ---- FM inference (daisy/model/FMRecommender.py:99-131): MF's kernels with score += (u_bias[u] + i_bias[c]) + bias_
extern "C" int drb_fm_rank(const float *d_P, const float *d_Q, const float *d_bias, int32_t U, int32_t I, int32_t F,
                           const int64_t *d_users, int64_t n_users, const int64_t *d_cands, int32_t cand_num, int32_t topk,
                           float *d_out, void *stream)
{
    DRB_REQUIRE(d_cands && d_out && d_bias && U > 0 && I > 0, "fm_rank: bad arguments");
    return launch_rank(0, d_P, d_Q, F, d_users, n_users, d_cands, cand_num, topk, d_out, nullptr, (cudaStream_t)stream, d_bias,
                       U, I);
}

extern "C" int drb_fm_full_rank(const float *d_P, const float *d_Q, const float *d_bias, int32_t U, int32_t I, int32_t F,
                                const int64_t *d_users, int64_t n_users, int32_t topk, int64_t *d_out, void *stream)
{
    DRB_REQUIRE(d_out && d_bias && U > 0 && I > 0, "fm_full_rank: bad arguments");
    return launch_rank(1, d_P, d_Q, F, d_users, n_users, nullptr, I, topk, nullptr, d_out, (cudaStream_t)stream, d_bias, U, I);
}

extern "C" int drb_fm_predict(const float *d_P, const float *d_Q, const float *d_bias, int32_t U, int32_t I, int32_t F,
                              const int32_t *d_u, const int32_t *d_i, int64_t n, float *d_out, void *stream)
{
    DRB_REQUIRE(d_bias && U > 0 && I > 0, "fm_predict: bad arguments");
    return launch_predict(d_P, d_Q, F, d_u, d_i, n, d_out, stream, d_bias, U, I);
}

extern "C" int drb_mf_rank_host(const float *d_P, const float *d_Q, int32_t F, const int64_t *h_users, int64_t n_users,
                                const int64_t *h_cands, int32_t cand_num, int32_t topk, float *h_out)
{
    DRB_REQUIRE(h_users && h_cands && h_out && n_users >= 0 && cand_num > 0 && topk > 0, "mf_rank_host: bad arguments");
    if (n_users == 0) return DRB_OK;
    int64_t *d_users = nullptr, *d_cands = nullptr;
    float *d_out = nullptr;
    size_t cb = sizeof(int64_t) * (size_t)n_users * cand_num, ob = sizeof(float) * (size_t)n_users * topk;
    DRB_CUDA(cudaMalloc((void **)&d_users, sizeof(int64_t) * (size_t)n_users));
    cudaError_t e = cudaMalloc((void **)&d_cands, cb);
    if (e == cudaSuccess) e = cudaMalloc((void **)&d_out, ob);
    if (e == cudaSuccess) e = cudaMemcpy(d_users, h_users, sizeof(int64_t) * (size_t)n_users, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(d_cands, h_cands, cb, cudaMemcpyHostToDevice);
    int rc = DRB_OK;
    if (e == cudaSuccess) rc = drb_mf_rank(d_P, d_Q, F, d_users, n_users, d_cands, cand_num, topk, d_out, nullptr);
    if (e == cudaSuccess && rc == DRB_OK) e = cudaMemcpy(h_out, d_out, ob, cudaMemcpyDeviceToHost);
    cudaFree(d_users); cudaFree(d_cands); cudaFree(d_out);
    if (e != cudaSuccess) return cuda_fail(e, "mf_rank_host", __FILE__, __LINE__);
    return rc;
}
