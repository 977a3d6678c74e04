// metrics.cu -- ranking KPIs of daisyRec's evaluation step on the device.
//
// Stands behind calc_ranking_results / Metric.run (daisy/utils/metrics.py:18-57, :59-96): for every
// cut-off K in common_ks the reference walks the test users in Python and calls np.in1d per user and
// per metric (:148-251).  Here ONE launch reads rank()'s float32 [n_users, topk] output where it
// already lies in HBM and produces every (cut-off, KPI) pair:
//   * one warp per test user, lane l owns list positions l, l+32, ...; a hit is a binary search of
//     the id in the user's sorted ground-truth CSR row (in1d semantics: duplicate ids each count);
//   * hit counts / first hit come from warp ballots, DCG and average-precision terms are summed in
//     fp64 with a fixed xor-butterfly, IDCG is a prefix table of 1/log2(k+2) in shared memory;
//   * per-user values are accumulated in a fixed order (warp -> CTA -> grid partials, then one
//     sequential pass), so results are bitwise reproducible run to run; fp64 throughout like the
//     reference (numpy float64).  np.mean sums pairwise, so parity is ~1e-15 relative (tested 1e-12);
//   * Coverage (:98-102) is a bitmap over item ids per cut-off, popcounted by the finishing kernel;
//   * Popularity (:104-122) sums item_pop over the UNIQUE hit ids (intersect1d) of the list.
// Traffic: n*topk*4 B of ids + the ground-truth rows; the kernel is latency, not bandwidth, bound.
#include "common.cuh"

namespace drb {

constexpr int KPI_N = DRB_KPI_COUNT;  // 8 values per cut-off
constexpr int KPI_MAXK = 8;           // cut-offs per launch
constexpr int KPI_MAXLD = 256;        // longest rank list
constexpr int KPI_WARPS = 8;
constexpr int KPI_SLOTS = KPI_MAXK * KPI_N;  // 64 accumulators, two per lane

struct KpiParams {
    const float *preds;
    long long n;
    int ld;
    const int64_t *gt_ptr;
    const int32_t *gt_idx;
    int ks[KPI_MAXK];
    int nk, kmax;
    int item_num;
    const double *item_pop;
    uint32_t *bitmap;   // [nk][words]
    long long words;
    double *partial;    // [grid][KPI_SLOTS]
};

__global__ void __launch_bounds__(KPI_WARPS * 32) kpi_kernel(KpiParams p)
{
    __shared__ double disc[KPI_MAXLD];          // 1 / log2(k + 2)
    __shared__ double cumdisc[KPI_MAXLD + 1];   // IDCG of h hits = sum_{t<h} disc[t]
    __shared__ double sval[KPI_WARPS][KPI_SLOTS];
    __shared__ int sid[KPI_WARPS][KPI_MAXLD];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int t = threadIdx.x; t < p.kmax; t += blockDim.x) disc[t] = 1.0 / log2((double)(t + 2));
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        cumdisc[0] = 0.0;
        for (int t = 0; t < p.kmax; ++t) {
            s += disc[t];
            cumdisc[t + 1] = s;
        }
    }
    __syncthreads();

    double acc0 = 0.0, acc1 = 0.0;  // slots lane and lane + 32
    const long long wglobal = (long long)blockIdx.x * KPI_WARPS + warp, wtotal = (long long)gridDim.x * KPI_WARPS;
    const int nchunk = (p.kmax + 31) >> 5;
    for (long long u = wglobal; u < p.n; u += wtotal) {
        const long long b = p.gt_ptr[u], ngt = p.gt_ptr[u + 1] - b;
        const int32_t *gt = p.gt_idx + b;
        const float *row = p.preds + u * (long long)p.ld;
        double dcg[KPI_MAXK], ap[KPI_MAXK], pop[KPI_MAXK];
        int hits[KPI_MAXK];
#pragma unroll
        for (int q = 0; q < KPI_MAXK; ++q) dcg[q] = ap[q] = pop[q] = 0.0, hits[q] = 0;
        int first = -1, carry = 0;
        uint32_t hmask[KPI_MAXLD / 32];
#pragma unroll
        for (int c = 0; c < KPI_MAXLD / 32; ++c) hmask[c] = 0u;
#pragma unroll
        for (int c = 0; c < KPI_MAXLD / 32; ++c) {
            if (c < nchunk) {
                const int pos = c * 32 + lane;
                const bool valid = pos < p.kmax;
                const float f = valid ? __ldg(row + pos) : -1.0f;
                const int v = (int)f;
                const bool isid = valid && v >= 0 && (float)v == f;  // in1d compares by value: only whole ids can hit
                bool hit = false;
                if (isid) {
                    long long lo = 0, hi = ngt;
                    while (lo < hi) {
                        long long mid = (lo + hi) >> 1;
                        if (__ldg(gt + mid) < v) lo = mid + 1; else hi = mid;
                    }
                    hit = lo < ngt && __ldg(gt + lo) == v;
                }
                sid[warp][pos] = isid ? v : -1 - pos;  // distinct negatives never compare equal
                const uint32_t hm = __ballot_sync(0xffffffffu, hit);
                hmask[c] = hm;
                const int cum = carry + __popc(hm & (0xffffffffu >> (31 - lane)));
                const double d = hit ? disc[pos] : 0.0, a = hit ? (double)cum / (double)(pos + 1) : 0.0;
#pragma unroll
                for (int q = 0; q < KPI_MAXK; ++q) {
                    if (q < p.nk) {
                        const int lim = p.ks[q] - c * 32;                   // positions of this chunk below the cut-off
                        const uint32_t m = lim >= 32 ? 0xffffffffu : lim <= 0 ? 0u : (1u << lim) - 1u;
                        hits[q] += __popc(hm & m);
                        if (pos < p.ks[q]) {
                            dcg[q] += d;
                            ap[q] += a;
                            if (isid && v < p.item_num) atomicOr(p.bitmap + q * p.words + (v >> 5), 1u << (v & 31));
                        }
                    }
                }
                if (first < 0 && hm) first = c * 32 + __ffs(hm) - 1;
                carry += __popc(hm);
            }
        }
        if (p.item_pop != nullptr) {  // sum over unique hit ids: a hit counts at its first occurrence only
            __syncwarp();
#pragma unroll
            for (int c = 0; c < KPI_MAXLD / 32; ++c) {
                if (c < nchunk) {
                    const int pos = c * 32 + lane;
                    if ((hmask[c] >> lane) & 1u) {
                        const int v = sid[warp][pos];
                        bool dup = false;
                        for (int j = 0; j < pos; ++j) dup |= sid[warp][j] == v;
                        if (!dup) {
                            const double w = __ldg(p.item_pop + v);
#pragma unroll
                            for (int q = 0; q < KPI_MAXK; ++q)
                                if (q < p.nk && pos < p.ks[q]) pop[q] += w;
                        }
                    }
                }
            }
        }
#pragma unroll
        for (int q = 0; q < KPI_MAXK; ++q) {
            if (q < p.nk) {
                const double sd = warp_sum(dcg[q]), sa = warp_sum(ap[q]), sp = warp_sum(pop[q]);
                if (lane == 0) {
                    const int h = hits[q];
                    const double idcg = cumdisc[h < p.kmax ? h : p.kmax];
                    double *o = &sval[warp][q * KPI_N];
                    o[DRB_KPI_RECALL] = (double)h / (double)ngt;
                    o[DRB_KPI_MRR] = (first >= 0 && first < p.ks[q]) ? 1.0 / (double)(first + 1) : 0.0;
                    o[DRB_KPI_NDCG] = idcg != 0.0 ? sd / idcg : 0.0;
                    o[DRB_KPI_HIT] = h ? 1.0 : 0.0;
                    o[DRB_KPI_PRECISION] = (double)h / (double)p.ks[q];
                    o[DRB_KPI_MAP] = h ? sa / (double)h : 0.0;
                    o[DRB_KPI_COVERAGE] = 0.0;
                    o[DRB_KPI_POPULARITY] = h ? sp / (double)ngt : 0.0;
                }
            }
        }
        __syncwarp();
        if (lane < p.nk * KPI_N) acc0 += sval[warp][lane];
        if (lane + 32 < p.nk * KPI_N) acc1 += sval[warp][lane + 32];
        __syncwarp();
    }
    // CTA partial: warps summed in index order
    __syncthreads();
    sval[warp][lane] = acc0;
    sval[warp][lane + 32] = acc1;
    __syncthreads();
    if (threadIdx.x < KPI_SLOTS) {
        double s = 0.0;
        for (int w = 0; w < KPI_WARPS; ++w) s += sval[w][threadIdx.x];
        p.partial[(long long)blockIdx.x * KPI_SLOTS + threadIdx.x] = s;
    }
}

// grid partials -> means (sequential, fixed order); bitmap -> coverage
__global__ void kpi_finish_kernel(KpiParams p, int grid, double *out)
{
    __shared__ unsigned long long cnt[KPI_MAXK];
    if (threadIdx.x < KPI_MAXK) cnt[threadIdx.x] = 0ull;
    __syncthreads();
    for (int q = 0; q < p.nk; ++q) {
        unsigned long long c = 0;
        for (long long w = threadIdx.x; w < p.words; w += blockDim.x) c += __popc(p.bitmap[q * p.words + w]);
        if (c) atomicAdd(&cnt[q], c);
    }
    __syncthreads();
    if (threadIdx.x < p.nk * KPI_N) {
        double s = 0.0;
        for (int b = 0; b < grid; ++b) s += p.partial[(long long)b * KPI_SLOTS + threadIdx.x];
        const int q = threadIdx.x / KPI_N, m = threadIdx.x - q * KPI_N;
        double v = s / (double)p.n;  // n == 0: 0/0 = NaN, like np.mean([])
        if (m == DRB_KPI_COVERAGE) v = (double)cnt[q] / (double)p.item_num;
        if (m == DRB_KPI_POPULARITY && p.item_pop == nullptr) v = 0.0;
        out[threadIdx.x] = v;
    }
}

static long long kpi_words(int item_num) { return ((long long)item_num + 31) / 32; }

}  // namespace drb

using namespace drb;

extern "C" size_t drb_rank_metrics_workspace_bytes(int32_t item_num, int32_t nk)
{
    if (item_num <= 0 || nk <= 0 || nk > KPI_MAXK) return 0;
    size_t bitmap = (size_t)nk * (size_t)kpi_words(item_num) * sizeof(uint32_t);
    bitmap = (bitmap + 255) & ~(size_t)255;
    return bitmap + (size_t)sm_count() * 4 * KPI_SLOTS * sizeof(double);
}

extern "C" int drb_rank_metrics(const float *d_preds, int64_t n_users, int32_t ld, const int64_t *d_gt_ptr,
                                const int32_t *d_gt_idx, const int32_t *h_ks, int32_t nk, int32_t item_num,
                                const double *d_item_pop, void *d_ws, double *d_out, void *stream)
{
    DRB_REQUIRE(d_out && h_ks && d_ws, "rank_metrics: null argument");
    DRB_REQUIRE(n_users >= 0 && (n_users == 0 || (d_preds && d_gt_ptr)), "rank_metrics: null inputs");
    DRB_REQUIRE(nk >= 1 && nk <= KPI_MAXK, "rank_metrics: 1..%d cut-offs per call, got %d", KPI_MAXK, nk);
    DRB_REQUIRE(ld >= 1 && item_num >= 1, "rank_metrics: bad list length %d / item_num %d", ld, item_num);
    KpiParams p{};
    p.kmax = 0;
    for (int q = 0; q < nk; ++q) {
        DRB_REQUIRE(h_ks[q] >= 1 && h_ks[q] <= ld && h_ks[q] <= KPI_MAXLD,
                    "rank_metrics: cut-off %d outside [1, min(list length %d, %d)]", h_ks[q], ld, KPI_MAXLD);
        p.ks[q] = h_ks[q];
        if (h_ks[q] > p.kmax) p.kmax = h_ks[q];
    }
    cudaStream_t st = (cudaStream_t)stream;
    p.preds = d_preds; p.n = n_users; p.ld = ld; p.gt_ptr = d_gt_ptr; p.gt_idx = d_gt_idx; p.nk = nk;
    p.item_num = item_num; p.item_pop = d_item_pop; p.words = kpi_words(item_num);
    size_t bitmap_bytes = ((size_t)nk * (size_t)p.words * sizeof(uint32_t) + 255) & ~(size_t)255;
    p.bitmap = (uint32_t *)d_ws;
    p.partial = (double *)((char *)d_ws + bitmap_bytes);
    DRB_CUDA(cudaMemsetAsync(p.bitmap, 0, bitmap_bytes, st));
    const int grid = grid_for(n_users, KPI_WARPS, 4);   // 4 per SM: the workspace holds sm_count() * 4 partial rows
    kpi_kernel<<<grid, KPI_WARPS * 32, 0, st>>>(p);
    DRB_CUDA(cudaGetLastError());
    kpi_finish_kernel<<<1, 256, 0, st>>>(p, grid, d_out);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}

extern "C" int drb_rank_metrics_host(const float *h_preds, int64_t n_users, int32_t ld, const int64_t *h_gt_ptr,
                                     const int32_t *h_gt_idx, const int32_t *h_ks, int32_t nk, int32_t item_num,
                                     const double *h_item_pop, double *h_out)
{
    DRB_REQUIRE(h_out && h_ks && n_users >= 0 && (n_users == 0 || (h_preds && h_gt_ptr)), "rank_metrics_host: null argument");
    DRB_REQUIRE(nk >= 1 && nk <= KPI_MAXK && ld >= 1 && item_num >= 1, "rank_metrics_host: bad arguments");
    const int64_t nnz = n_users ? h_gt_ptr[n_users] : 0;
    DRB_REQUIRE(nnz == 0 || h_gt_idx, "rank_metrics_host: null ground truth");
    float *d_preds = nullptr;
    int64_t *d_ptr = nullptr;
    int32_t *d_idx = nullptr;
    double *d_pop = nullptr, *d_out = nullptr;
    void *d_ws = nullptr;
    cudaStream_t st = nullptr;
    int rc = DRB_OK;
    cudaError_t e = cudaSuccess;
    auto ok = [&](cudaError_t r) { if (e == cudaSuccess) e = r; return e == cudaSuccess; };
    const size_t pb = sizeof(float) * (size_t)(n_users * ld), tb = sizeof(int64_t) * (size_t)(n_users + 1);
    ok(cudaMalloc(&d_preds, pb ? pb : 4)) && ok(cudaMalloc(&d_ptr, tb)) &&
        ok(cudaMalloc(&d_idx, nnz ? sizeof(int32_t) * (size_t)nnz : 4)) &&
        ok(cudaMalloc(&d_out, sizeof(double) * KPI_SLOTS)) &&
        ok(cudaMalloc(&d_ws, drb_rank_metrics_workspace_bytes(item_num, nk)));
    if (h_item_pop) ok(cudaMalloc(&d_pop, sizeof(double) * (size_t)item_num));
    if (e == cudaSuccess) {
        if (pb) ok(cudaMemcpyAsync(d_preds, h_preds, pb, cudaMemcpyHostToDevice, st));
        if (n_users) ok(cudaMemcpyAsync(d_ptr, h_gt_ptr, tb, cudaMemcpyHostToDevice, st));
        else ok(cudaMemsetAsync(d_ptr, 0, tb, st));
        if (nnz) ok(cudaMemcpyAsync(d_idx, h_gt_idx, sizeof(int32_t) * (size_t)nnz, cudaMemcpyHostToDevice, st));
        if (h_item_pop) ok(cudaMemcpyAsync(d_pop, h_item_pop, sizeof(double) * (size_t)item_num, cudaMemcpyHostToDevice, st));
    }
    if (e == cudaSuccess) {
        rc = drb_rank_metrics(d_preds, n_users, ld, d_ptr, d_idx, h_ks, nk, item_num, d_pop, d_ws, d_out, st);
        if (rc == DRB_OK) {
            ok(cudaMemcpyAsync(h_out, d_out, sizeof(double) * (size_t)nk * KPI_N, cudaMemcpyDeviceToHost, st));
            ok(cudaStreamSynchronize(st));
        }
    }
    cudaFree(d_preds); cudaFree(d_ptr); cudaFree(d_idx); cudaFree(d_pop); cudaFree(d_out); cudaFree(d_ws);
    if (e != cudaSuccess) return cuda_fail(e, "rank_metrics_host", __FILE__, __LINE__);
    return rc;
}
