// mf_bpr.cu -- the BPR-MF training step as ONE persistent cooperative sm_90a kernel.
//
// Stands behind GeneralRecommender.fit's step loop (daisy/model/AbstractRecommender.py:112-128)
// with MF.calc_loss (daisy/model/MFRecommender.py:70-97), BPRLoss (daisy/utils/loss.py:11),
// autograd's embedding backward (:125) and optim.SGD/Adam.step (:126, :53-56).
//
// Synchronous-step semantics (every gradient of a step is taken at the PRE-step weights, the
// Frobenius norms couple the whole batch) are kept exactly, without ever materialising the
// reference's table-sized dense gradient:
//
//   phase 1 (read-only on P,Q)   per triple (u,i,j): index tile staged by TMA (cp.async.bulk) into
//       shared memory; a group of W lanes gathers the three factor rows with 128-bit L2 loads,
//       reduces the two dot products with xor-shuffles (canonical order), evaluates
//       s = sigmoid(x), loss = -log(1e-10+s), c = -s(1-s)/(1e-10+s) and issues vector
//       RED.ADD.F32x4 reductions of the BPR part of the gradient into the L2-resident
//       accumulators gP/gQ:  gP[u] += c(q_i-q_j), gQ[i] += c p_u, gQ[j] -= c p_u; it also counts how
//       often each row occurs (cntU, cntI = pos | neg<<32) and accumulates the six batch norms.
//   -- grid barrier --           (norms and loss are now final; nobody reads P,Q any more)
//   phase 2                      every touched row is applied exactly once:
//       g = gP[r] + cnt * (reg_1 sgn(theta) + reg_2 theta / ||.||_F);  theta -= lr g  (or Adam);
//       the accumulator row and its counter are reset for the next step.  Rows are found either
//       by a dense sweep (large batches: every row is touched) or by claiming the counter with
//       atomicExch from the triple that touched it (small batches).
//   -- grid barrier --           next step.
//
// A NaN loss (ValueError in the reference, :122-123) stops the loop before the update of that step.
//
// Variants of the same kernel: GEN = false is the BPR-only hot instantiation, GEN = true selects HingeLoss / TOP1Loss
// (daisy/utils/loss.py:16-33) or the point-wise CL / SL branch (MFRecommender.py:75-81: the third plane holds the label,
// only P_u and Q_i take part) at run time; `phases` splits it into phase-1 / phase-2 launches (multi-GPU exchange,
// LightGCN, NeuMF); `neg_row_ptr` switches on the fused sampler (a fresh negative per triple drawn inside phase 1).
#include <math.h>
#include <stdlib.h>

#include <atomic>
#include <map>
#include <mutex>
#include <vector>

#include "step_kernel.cuh"

namespace drb {

// b?[k] = triples[perm[k], ?]
__global__ void gather_triples_kernel(const int32_t *__restrict__ triples, const int64_t *__restrict__ perm, long long n,
                                      int32_t *__restrict__ bu, int32_t *__restrict__ bi, int32_t *__restrict__ bj)
{
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
        long long src = perm ? perm[k] : k;
        const int32_t *t = triples + 3 * src;
        bu[k] = __ldg(t);
        bi[k] = __ldg(t + 1);
        bj[k] = __ldg(t + 2);
    }
}

// ------------------------------------------------------------------ host dispatch
typedef void (*StepKernel)(StepParams);

template <int VEC, bool GEN>
static StepKernel pick_kernel_v(int W, int NCH)
{
#define DRB_CASE(w, n) \
    if (W == w && NCH == n) return mf_bpr_steps_kernel<VEC, w, n, GEN>;
    DRB_CASE(1, 1) DRB_CASE(2, 1) DRB_CASE(4, 1) DRB_CASE(8, 1) DRB_CASE(16, 1) DRB_CASE(32, 1)
    DRB_CASE(32, 2) DRB_CASE(32, 4) DRB_CASE(32, 8)
#undef DRB_CASE
    return nullptr;
}

// The lean MF instantiation.  Its lane geometry is its own: the index loads, address arithmetic, loss chain and counter updates
// of a triple are replayed by every lane of the row's group, the row arithmetic is not -- so fewer lanes per row (more chunks of
// 4 floats per lane) means fewer issue slots per triple and more rows in flight per warp.  Candidates for a factor count are
// every (W lanes, NCH in {4, 2, 1} chunks per lane) with W a power of two; the preferred one keeps 8 lanes per row, so that one
// 128-bit access of a group still covers exactly one 128-byte line (F = 64: 8 lanes x 2 chunks, F = 128: 8 x 4).  Which
// candidate runs is decided on the device (lean_autotune).  Only the fp32 summation order of the two dot products differs from
// the canonical geometry (row_geom) that rank / predict / the oracle share.
static int lean_nch_only()
{
    static const int v = [] {
        const char *e = getenv("DRB_LEAN_NCH");   // developer switch: restrict the candidates to 1 | 2 | 4 chunks per lane
        int n = e ? atoi(e) : 0;
        return (n == 1 || n == 2 || n == 4) ? n : 0;
    }();
    return v;
}
// candidates in order of preference; returns their number (at most 3)
static int lean_candidates(int F, int (&cw)[3], int (&cn)[3])
{
    int count = 0;
    if (F <= 0 || F % 4 != 0) return 0;
    const int chunks = F / 4;
    auto valid = [&](int n) {
        if (chunks % n != 0) return false;
        const int w = chunks / n;
        return w <= 32 && (w & (w - 1)) == 0;
    };
    auto push = [&](int n) {
        for (int k = 0; k < count; ++k) if (cn[k] == n) return;
        if (lean_nch_only() != 0 && n != lean_nch_only()) return;
        cw[count] = chunks / n;
        cn[count] = n;
        ++count;
    };
    for (int n = 4; n >= 1; n >>= 1)                       // preferred: the most chunks per lane that keep whole lines (W >= 8)
        if (valid(n) && (chunks / n >= 8 || n == 1)) { push(n); break; }
    for (int n = 4; n >= 1; n >>= 1)
        if (valid(n)) push(n);
    if (count == 0 && lean_nch_only() == 0) {              // e.g. F = 100: 25 chunks on 32 lanes
        RowGeom g = row_geom(F);
        if (g.vec == 4 && g.nch == 1) { cw[0] = g.width; cn[0] = 1; count = 1; }
    }
    return count;
}
void lean_default_geom(int F, int &W, int &NCH)            // host-only: the preferred candidate
{
    int cw[3], cn[3];
    W = NCH = 0;
    if (lean_candidates(F, cw, cn) > 0) { W = cw[0]; NCH = cn[0]; }
}
static StepKernel pick_lean_wn(int W, int NCH)
{
#define DRB_LEAN(w, n) \
    if (W == w && NCH == n) return mf_bpr_steps_lean_kernel<4, w, n>;
    DRB_LEAN(1, 1) DRB_LEAN(2, 1) DRB_LEAN(4, 1) DRB_LEAN(8, 1) DRB_LEAN(16, 1) DRB_LEAN(32, 1)
    DRB_LEAN(1, 2) DRB_LEAN(2, 2) DRB_LEAN(4, 2) DRB_LEAN(8, 2) DRB_LEAN(16, 2) DRB_LEAN(32, 2)
    DRB_LEAN(1, 4) DRB_LEAN(2, 4) DRB_LEAN(4, 4) DRB_LEAN(8, 4) DRB_LEAN(16, 4) DRB_LEAN(32, 4)
#undef DRB_LEAN
    return nullptr;
}
// the user-bucketed mode of the lean kernel: instantiated for the preferred geometries of F = 32 and 64 (8 lanes x 1 or 2 chunks);
// at 8 x 4 (F = 128) it spills under the 128-register bound of two resident CTAs per SM
static StepKernel pick_lean_ub(int W, int NCH)
{
    if (W != 8) return nullptr;
    if (NCH == 1) return mf_bpr_steps_lean_kernel<4, 8, 1, true>;
    if (NCH == 2) return mf_bpr_steps_lean_kernel<4, 8, 2, true>;
    return nullptr;
}
// its staged SGD form (user rows staged per bucket, tiles sorted by user, item regulariser per occurrence): its own
// instantiation, so that neither form carries the other's registers; launch_kernel swaps it in when the launch can stage
static StepKernel staged_twin(StepKernel k)
{
    if (k == mf_bpr_steps_lean_kernel<4, 8, 1, true>) return mf_bpr_steps_lean_kernel<4, 8, 1, true, true>;
    if (k == mf_bpr_steps_lean_kernel<4, 8, 2, true>) return mf_bpr_steps_lean_kernel<4, 8, 2, true, true>;
    return nullptr;
}
static int ubucket_switch()
{
    static const int v = [] {
        const char *e = getenv("DRB_UBUCKET");   // developer switch: 0 forbids the user-bucketed mode, 1 forces it (once checked)
        return e ? (atoi(e) != 0 ? 1 : 0) : -1;
    }();
    return v;
}

// Users per bucket of the user-bucketed mode: about 8 buckets per resident CTA, so that the dynamic claiming of buckets balances
// the phase (bucket sizes follow the user degrees); at least kUbMinUsers, at most what a 64 KB shared accumulator holds and
// kUbMaxRows (the keys of the per-tile user sort).  0 when the mode cannot run the problem (more than kUbMaxBuckets buckets: the
// per-CTA histogram would not fit shared memory).
constexpr int kUbMinUsers = 16, kUbMaxBuckets = 8192;
// dynamic shared memory the staged SGD user side may take (two CTAs per SM keep fitting next to the 39 KB of static index tiles
// and per-tile sort arrays): 51 KB at F = 64 and 66 users per bucket (ML-20M on 132 SMs); it stages up to 84 users per bucket at
// F = 64, 168 at F = 32
constexpr size_t kUbStagedSmem = 65536;
constexpr long long kUbTimedBatch = 1 << 19;   // triples per step of the on-device timing problem (lean_autotune)
static int ub_users_for(int U, int F, long long batch)
{
    const int target = 8 * DRB_MINB * sm_count();
    int ub = (U + target - 1) / target;
    if (ub < kUbMinUsers) ub = kUbMinUsers;
    const int cap = 65536 / ((F + 1) * 4 + 4);   // width rule: F + 1 floats and a counter per user (the accumulator takes F)
    if (ub > cap) ub = cap;
    if (ub > kUbMaxRows) ub = kUbMaxRows;
    if (ub < 1) return 0;
    const long long nbk = ((long long)U + ub - 1) / ub;
    return (nbk <= kUbMaxBuckets && batch + 4 * nbk < (1LL << 31)) ? ub : 0;
}
// SGD stages the bucket's user rows (two slots: the current bucket's and the prefetched next one's) next to the accumulator of
// `ub` users, when both fit kUbStagedSmem (ub (12 F + 4) bytes); wider buckets keep the accumulate-then-sweep user side
static bool ub_staged(const StepParams &p, int ub)
{
    const size_t acc = sizeof(float) * (size_t)ub * p.F + sizeof(unsigned) * ub;
    const size_t rows = 2 * sizeof(float) * (size_t)ub * p.F;
    return p.opt == DRB_OPT_SGD && p.gscale == 1.f && p.neg_mult == 1.f && acc + rows <= kUbStagedSmem;
}

// The bucketed mode's scratch (counters, bucket ranges, user and item norm cache, partitioned triples): library-owned, grow-only,
// one per device and stream; it depends on the batch, so it cannot live in the workspace.  Its counters are cleared before every
// launch, the norm cache (staged SGD mode only) is filled by the launch itself.  Each buffer lives as long as the process: about
// 16 B x the largest batch of bucketed steps launched on that stream + 8 B per user and item (18.1 MB at B = 1 M and ML-20M), so a
// caller that trains on many streams holds one such buffer per stream.
static int ub_scratch(StepParams &p, cudaStream_t st, bool staged)
{
    static std::mutex mu;
    static std::map<std::pair<int, cudaStream_t>, std::pair<void *, size_t>> bufs;
    const size_t nbk = (size_t)p.ub_buckets;
    const size_t cnt_b = align256(sizeof(unsigned) * (2 * nbk + 1)), rng_b = align256(sizeof(int) * 2 * nbk);
    const size_t nrm_b = staged ? align256(sizeof(float2) * ((size_t)p.U + p.I)) : 0;
    const size_t need = cnt_b + rng_b + nrm_b + sizeof(int4) * (size_t)p.batch;
    int dev = 0;
    DRB_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lock(mu);
    auto &e = bufs[std::make_pair(dev, st)];
    if (e.second < need) {
        if (e.first != nullptr) {
            DRB_CUDA(cudaStreamSynchronize(st));   // an earlier launch on this stream may still read it
            DRB_CUDA(cudaFree(e.first));
            e = std::make_pair(nullptr, (size_t)0);
        }
        DRB_CUDA(cudaMalloc(&e.first, need));
        e.second = need;
    }
    char *b = (char *)e.first;
    p.ub_count = (unsigned *)b;
    p.ub_range = (int *)(b + cnt_b);
    p.ub_norm = staged ? (float2 *)(b + cnt_b + rng_b) : nullptr;
    p.ub_t = (int4 *)(b + cnt_b + rng_b + nrm_b);
    DRB_CUDA(cudaMemsetAsync(p.ub_count, 0, sizeof(unsigned) * (2 * nbk + 1), st));
    return DRB_OK;
}

// GEN = false: BPR only (the hot instantiation, no loss-kind branches); GEN = true: HL / TL selected at run time
static StepKernel pick_kernel(int F, bool gen)
{
    if (F <= 0) return nullptr;
    RowGeom g = row_geom(F);
    if (gen) {
        if (g.vec == 4) return pick_kernel_v<4, true>(g.width, g.nch);
        if (g.vec == 2) return pick_kernel_v<2, true>(g.width, g.nch);
        return pick_kernel_v<1, true>(g.width, g.nch);
    }
    if (g.vec == 4) return pick_kernel_v<4, false>(g.width, g.nch);
    if (g.vec == 2) return pick_kernel_v<2, false>(g.width, g.nch);
    return pick_kernel_v<1, false>(g.width, g.nch);
}

// grid / tile choice and the cooperative launch of one chosen instantiation
// (ub: k is a user-bucketed instantiation; the launch sizes its buckets, scratch and dynamic shared memory)
static int launch_kernel(StepKernel k, StepParams &p, cudaStream_t st, bool keep_status, int tile_cap = kTileDefault,
                         bool ub = false)
{
    size_t smem = 0;
    if (ub) {
        p.ub_users = ub_users_for(p.U, p.F, p.batch);
        DRB_REQUIRE(p.ub_users > 0, "user-bucketed step: %d users in more than %d buckets", p.U, kUbMaxBuckets);
        p.ub_buckets = (p.U + p.ub_users - 1) / p.ub_users;
        // staged form (ub_staged) or accumulate-then-sweep (accumulator row stride: F staged, F + 1 otherwise; the staged form
        // adds the item regulariser once per occurrence in phase 1: unscaled gradients, one count per occurrence)
        const size_t acc = sizeof(float) * (size_t)p.ub_users * p.F + sizeof(unsigned) * p.ub_users;
        const size_t rows = 2 * sizeof(float) * (size_t)p.ub_users * p.F;
        const bool staged = ub_staged(p, p.ub_users);
        const size_t need = staged ? acc + rows : acc + sizeof(float) * (size_t)p.ub_users;
        const size_t hist = 2 * sizeof(unsigned) * (size_t)p.ub_buckets;
        smem = ((need > hist ? need : hist) + 15) / 16 * 16;
        const int rc = ub_scratch(p, st, staged);
        if (rc != DRB_OK) return rc;
        if (staged) k = staged_twin(k);
        DRB_REQUIRE(k != nullptr, "user-bucketed step: no staged instantiation");
    }
    // occupancy of the chosen instantiation, cached per device (the query costs microseconds and this runs once per step in the
    // split multi-GPU / LightGCN / NeuMF paths); the dynamic shared-memory limit is a per-device function attribute
    static thread_local StepKernel cached_k = nullptr;
    static thread_local size_t cached_smem = 0;
    static thread_local int cached_dev = -1, cached_per_sm = 0;
    int dev = 0;
    DRB_CUDA(cudaGetDevice(&dev));
    if (cached_k != k || cached_smem != smem || cached_dev != dev) {
        int q = 0;
        if (smem > 0) DRB_CUDA(cudaFuncSetAttribute((const void *)k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        DRB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&q, k, kThreads, smem));
        cached_k = k;
        cached_smem = smem;
        cached_dev = dev;
        cached_per_sm = q;
    }
    const int per_sm = cached_per_sm;
    DRB_REQUIRE(per_sm > 0, "step kernel does not fit on an SM");
    const int max_grid = per_sm * sm_count();
    // tile: equal tiles of at most kTileMax triples, every CTA the same number of them
    const int tile = pick_tile((p.batch + max_grid - 1) / max_grid, tile_cap);
    p.tile = tile;
    long long tiles = (p.batch + tile - 1) / tile;
    long long rows_work = ((long long)p.U + p.I + 63) / 64;
    bool dense = p.dense_hint >= 0 ? (p.dense_hint != 0)
                                   : ((p.opt != DRB_OPT_SGD) || (3 * p.batch >= ((long long)p.U + p.I) / 4));
    long long want_grid = (dense && p.apply) ? (tiles > rows_work ? tiles : rows_work) : tiles;
    int grid = (int)(want_grid < 1 ? 1 : (want_grid > max_grid ? max_grid : want_grid));
    if (p.phases & 1)
        DRB_CUDA(cudaMemsetAsync(p.ws.hdr, 0, (p.phases == 3 && !keep_status) ? sizeof(WsHeader) : kHdrResetBytes, st));
    void *args[] = {&p};
    DRB_CUDA(cudaLaunchCooperativeKernel((void *)k, dim3(grid), dim3(kThreads), args, smem, st));
    return DRB_OK;
}

// ---- on-device selection of the step instantiation (lean_autotune below): seeded problems built on the host
struct CheckProblem {
    int U, I, F, B, K;
    std::vector<float> hP, hQ;
    std::vector<int32_t> hu, hi, hj;
};
static void make_check_problem(CheckProblem &c, int U, int I, int F, int B, int K, bool hot_users)
{
    c.U = U; c.I = I; c.F = F; c.B = B; c.K = K;
    c.hP.resize((size_t)U * F);
    c.hQ.resize((size_t)I * F);
    const long long n = (long long)B * K;
    c.hu.resize(n); c.hi.resize(n); c.hj.resize(n);
    unsigned long long x = 0x9E3779B97F4A7C15ull;
    auto rnd = [&]() { x = x * 6364136223846793005ull + 1442695040888963407ull; return (uint32_t)(x >> 33); };
    for (auto &v : c.hP) v = ((float)(rnd() % 20001) - 10000.f) * 2e-5f;
    for (auto &v : c.hQ) v = ((float)(rnd() % 20001) - 10000.f) * 2e-5f;
    for (long long t = 0; t < n; ++t) {
        c.hu[t] = (int32_t)(rnd() % (uint32_t)(hot_users ? U / 4 : U));
        const unsigned long long a = rnd() % (uint32_t)I;
        c.hi[t] = (int32_t)(hot_users ? a : a * a / (unsigned)I);      // timing problem: popular items, like the bench's planes
        c.hj[t] = (int32_t)(rnd() % (uint32_t)I);
    }
}
// one launch of K steps of instantiation k on a fresh copy of the problem; optional outputs: tables, losses, milliseconds of a
// second (warm) launch
static bool run_check_variant(const CheckProblem &c, StepKernel k, int opt, float lr, std::vector<float> *outP,
                              std::vector<float> *outQ, double *loss, float *ms, int tile_cap = kTileDefault, bool ub = false)
{
    const long long n = (long long)c.B * c.K;
    const size_t wsb = carve(nullptr, c.U, c.I, c.F, opt, nullptr);
    float *dP = nullptr, *dQ = nullptr;
    void *dws = nullptr;
    int32_t *du = nullptr, *di = nullptr, *dj = nullptr;
    double *dl = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    bool good = cudaMalloc(&dP, c.hP.size() * 4) == cudaSuccess && cudaMalloc(&dQ, c.hQ.size() * 4) == cudaSuccess &&
                cudaMalloc(&dws, wsb) == cudaSuccess && cudaMalloc(&du, n * 4) == cudaSuccess &&
                cudaMalloc(&di, n * 4) == cudaSuccess && cudaMalloc(&dj, n * 4) == cudaSuccess &&
                cudaMalloc(&dl, c.K * 8) == cudaSuccess && cudaEventCreate(&e0) == cudaSuccess &&
                cudaEventCreate(&e1) == cudaSuccess;
    if (good) {
        cudaMemcpy(dP, c.hP.data(), c.hP.size() * 4, cudaMemcpyHostToDevice);
        cudaMemcpy(dQ, c.hQ.data(), c.hQ.size() * 4, cudaMemcpyHostToDevice);
        cudaMemcpy(du, c.hu.data(), n * 4, cudaMemcpyHostToDevice);
        cudaMemcpy(di, c.hi.data(), n * 4, cudaMemcpyHostToDevice);
        cudaMemcpy(dj, c.hj.data(), n * 4, cudaMemcpyHostToDevice);
        cudaMemset(dws, 0, wsb);
        drb_hyper h = {lr, 0.001f, 0.001f, opt, 0.9f, 0.999f, 1e-8f, DRB_LOSS_BPR};
        StepParams p;
        good = fill_params(p, dP, dQ, dws, c.U, c.I, c.F, du, di, dj, n, c.B, 0, c.K, &h, 0, dl, 1) == DRB_OK &&
               launch_kernel(k, p, (cudaStream_t)0, false, tile_cap, ub) == DRB_OK &&
               cudaStreamSynchronize((cudaStream_t)0) == cudaSuccess;
        if (good && ms != nullptr) {
            *ms = 0.f;
            for (int rep = 0; rep < 2 && good; ++rep) {            // best of two warm launches
                float t = 0.f;
                cudaEventRecord(e0, (cudaStream_t)0);
                good = launch_kernel(k, p, (cudaStream_t)0, false, tile_cap, ub) == DRB_OK;
                cudaEventRecord(e1, (cudaStream_t)0);
                good = good && cudaEventSynchronize(e1) == cudaSuccess && cudaEventElapsedTime(&t, e0, e1) == cudaSuccess;
                if (good && (rep == 0 || t < *ms)) *ms = t;
            }
        }
    }
    if (good && outP != nullptr) {
        outP->resize(c.hP.size());
        outQ->resize(c.hQ.size());
        good = cudaMemcpy(outP->data(), dP, c.hP.size() * 4, cudaMemcpyDeviceToHost) == cudaSuccess &&
               cudaMemcpy(outQ->data(), dQ, c.hQ.size() * 4, cudaMemcpyDeviceToHost) == cudaSuccess &&
               cudaMemcpy(loss, dl, c.K * 8, cudaMemcpyDeviceToHost) == cudaSuccess;
    }
    cudaFree(dP); cudaFree(dQ); cudaFree(dws); cudaFree(du); cudaFree(di); cudaFree(dj); cudaFree(dl);
    if (e0) cudaEventDestroy(e0);
    if (e1) cudaEventDestroy(e1);
    return good;
}

// what the BPR + SGD / Adam steps of one factor count run with
struct LeanChoice {
    int W = 0, NCH = 0;               // lanes per row, chunks per lane of the lean instantiation; W == 0: the general one
    int tile_cap = kTileDefault;
    int ub_W = 0, ub_NCH = 0;         // geometry of the user-bucketed mode when it was selected (it then runs the fused steps)
    float ms_general = 0.f, ms_lean = 0.f;   // timed launch of the autotune (the lean kernel that runs: best lean candidate or
                                             // the bucketed mode)
};

// the user-bucketed mode's edge cases: several buckets, U not a multiple of the bucket width, an empty bucket (2), and one user
// with more triples in a step than an index tile holds (run at lr 0.01: at 0.05 its large item sums leave the fp32 noise of the
// general kernel alone near the 1e-5 table tolerance)
static void make_bucket_problem(CheckProblem &c, int F)
{
    make_check_problem(c, 5 * kUbMinUsers + 7, 64, F, 3000, 2, false);
    for (size_t t = 0; t < c.hu.size(); ++t) {
        if (t % 5 < 2) c.hu[t] = 3;                                           // 1 200 triples of user 3 per step
        else if (c.hu[t] / kUbMinUsers == 2) c.hu[t] += kUbMinUsers;
    }
}

// same losses (1e-5 rel) and tables (1e-5 abs) as the reference outputs of the general instantiation
static bool same_results(const CheckProblem &c, int opt, const std::vector<float> &P0, const std::vector<float> &Q0,
                         const double *l0, const std::vector<float> &P1, const std::vector<float> &Q1, const double *l1)
{
    bool ok = true;
    for (int k = 0; k < c.K; ++k) ok = ok && fabs(l0[k] - l1[k]) <= 1e-5 * fabs(l0[k]) && l0[k] > 0.0;
    // Adam turns a gradient that is pure rounding noise into a +-lr step of either sign: a few such elements may differ by up to
    // 2 lr between ANY two runs (also of the same kernel); everything else agrees to 1e-5
    int bad = 0;
    float worst = 0.f;
    double moved = 0.0;
    for (size_t e = 0; e < P0.size(); ++e) {
        const float dlt = fabsf(P0[e] - P1[e]);
        if (!(dlt <= 1e-5f)) { ++bad; worst = fmaxf(worst, dlt); }
        moved = fmax(moved, fabs((double)P0[e] - c.hP[e]));
    }
    for (size_t e = 0; e < Q0.size(); ++e) {
        const float dlt = fabsf(Q0[e] - Q1[e]);
        if (!(dlt <= 1e-5f)) { ++bad; worst = fmaxf(worst, dlt); }
    }
    ok = ok && (bad == 0 || (opt == DRB_OPT_ADAM && bad <= 4 && worst <= 0.11f));
    return ok && moved > 1e-4;                                   // and the steps did move the tables
}

// L2 size of the current device (the regime test and the L2-regime timing problem are sized from it)
static long long l2_bytes()
{
    static const long long l2 = [] {
        int dev = 0, bytes = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&bytes, cudaDevAttrL2CacheSize, dev) != cudaSuccess) {
            cudaGetLastError();
            bytes = 0;
        }
        return (long long)(bytes > 0 ? bytes : 64 << 20);
    }();
    return l2;
}

// Nothing about the speed of the lean instantiations is assumed: once per process, factor count and regime every candidate
// geometry (1) must reproduce the general instantiation on a small seeded problem (two SGD and two Adam steps), and (2) is
// timed against it on a problem of the caller's regime with the bench's index statistics (3 steps x 524 288 triples, best of
// two warm launches).  The fastest correct candidate is used if it beats the general
// instantiation, and a larger index tile if that helps it further; otherwise the general kernel stays.  Never a wrong table,
// never a slower step.
static LeanChoice lean_autotune(int F, bool hbm)
{
    LeanChoice best;
    StepKernel gen = pick_kernel(F, false);
    int cw[3], cn[3];
    const int ncand = lean_candidates(F, cw, cn);
    if (gen == nullptr || ncand == 0) return best;
    CheckProblem small, big;
    make_check_problem(small, 96, 80, F, 384, 2, true);
    // timing problem: for the L2 regime U = 4 I rows whose tables + accumulators take half of this device's L2 (the other half is
    // left to the streamed index planes); for the HBM regime 2 x 134 MB of user rows
    const long long l2_rows = l2_bytes() / (2LL * 8 * F) * 4 / 5;
    const int rows = hbm ? 33554432 / F : (int)(l2_rows > 4096 ? l2_rows : 4096);
    make_check_problem(big, rows, hbm ? 16384 : rows / 4, F, (int)kUbTimedBatch, 3, false);
    std::vector<float> refP[2], refQ[2];
    double refl[2][2];
    bool ok = true;
    for (int opt = DRB_OPT_SGD; opt <= DRB_OPT_ADAM && ok; ++opt)
        ok = run_check_variant(small, gen, opt, 0.05f, &refP[opt], &refQ[opt], refl[opt], nullptr);
    ok = ok && run_check_variant(big, gen, DRB_OPT_SGD, 0.01f, nullptr, nullptr, nullptr, &best.ms_general);
    float best_ms = 0.f;
    for (int k = 0; k < ncand && ok; ++k) {
        StepKernel lean = pick_lean_wn(cw[k], cn[k]);
        if (lean == nullptr) continue;
        bool same = true;
        for (int opt = DRB_OPT_SGD; opt <= DRB_OPT_ADAM && same; ++opt) {
            std::vector<float> P1, Q1;
            double l1[2];
            same = run_check_variant(small, lean, opt, 0.05f, &P1, &Q1, l1, nullptr) &&
                   same_results(small, opt, refP[opt], refQ[opt], refl[opt], P1, Q1, l1);
        }
        cudaGetLastError();
        if (!same) {
            fprintf(stderr, "[daisyrec_b200] lean step kernel %d lanes x %d chunks (factors=%d) did not reproduce the general "
                            "instantiation: not used\n", cw[k], cn[k], F);
            continue;
        }
        float ms = 0.f;
        if (!run_check_variant(big, lean, DRB_OPT_SGD, 0.01f, nullptr, nullptr, nullptr, &ms) || !(ms > 0.f)) continue;
        if (best_ms == 0.f || ms < best_ms) { best_ms = ms; best.W = cw[k]; best.NCH = cn[k]; }
    }
    cudaGetLastError();
    best.ms_lean = best_ms;
    if (!ok || best.W == 0 || !(best_ms < 0.98f * best.ms_general)) {
        if (ok && best.W != 0)
            fprintf(stderr, "[daisyrec_b200] lean step kernel (factors=%d): %.3f ms against %.3f ms of the general instantiation on "
                            "the timing problem: keeping the general one\n", F, best_ms, best.ms_general);
        best.W = best.NCH = 0;
    } else {
        float ms_big_tile = 0.f;                                  // a larger index tile for the chosen candidate?
        if (run_check_variant(big, pick_lean_wn(best.W, best.NCH), DRB_OPT_SGD, 0.01f, nullptr, nullptr, nullptr, &ms_big_tile,
                              kTileMax) && ms_big_tile > 0.f && ms_big_tile < 0.98f * best_ms) {
            best.tile_cap = kTileMax;
            best.ms_lean = ms_big_tile;
        }
        cudaGetLastError();
    }
    // The user-bucketed mode (preferred geometry): the same two checks on the small problem and on its edge-case problem, then
    // timed on the regime's problem; it runs if it beats what would run otherwise by 2 % (or DRB_UBUCKET=1).
    StepKernel ub = pick_lean_ub(cw[0], cn[0]);
    if (!ok || ub == nullptr || ubucket_switch() == 0) return best;
    CheckProblem edge;
    make_bucket_problem(edge, F);
    bool same = true;
    for (int opt = DRB_OPT_SGD; opt <= DRB_OPT_ADAM && same; ++opt) {
        std::vector<float> P0, Q0, P1, Q1;
        double l0[2], l1[2];
        same = run_check_variant(small, ub, opt, 0.05f, &P1, &Q1, l1, nullptr, kTileDefault, true) &&
               same_results(small, opt, refP[opt], refQ[opt], refl[opt], P1, Q1, l1) &&
               run_check_variant(edge, gen, opt, 0.01f, &P0, &Q0, l0, nullptr) &&
               run_check_variant(edge, ub, opt, 0.01f, &P1, &Q1, l1, nullptr, kTileDefault, true) &&
               same_results(edge, opt, P0, Q0, l0, P1, Q1, l1);
    }
    cudaGetLastError();
    if (!same) {
        fprintf(stderr, "[daisyrec_b200] user-bucketed step kernel (factors=%d) did not reproduce the general instantiation: not "
                        "used\n", F);
        return best;
    }
    float ms = 0.f;
    const bool timed = run_check_variant(big, ub, DRB_OPT_SGD, 0.01f, nullptr, nullptr, nullptr, &ms, best.tile_cap, true) &&
                       ms > 0.f;
    cudaGetLastError();
    const float current = best.W > 0 ? best.ms_lean : best.ms_general;
    if (timed && (ubucket_switch() == 1 || ms < 0.98f * current)) {
        best.ub_W = cw[0];
        best.ub_NCH = cn[0];
        best.ms_lean = ms;
    }
    return best;
}

// regime of a problem: do the two tables and their accumulators fit the L2 cache?
static bool hbm_regime(long long table_rows, int F)
{
    return table_rows * (long long)F * 8 > l2_bytes();
}

static const LeanChoice &lean_choice(int F, long long table_rows)
{
    static const bool no_lean = getenv("DRB_NO_LEAN") != nullptr;   // developer switch: A/B the instantiations
    static std::mutex mu;
    static std::map<int, LeanChoice> state;
    const bool hbm = hbm_regime(table_rows, F);
    const int key = F * 2 + (hbm ? 1 : 0);
    std::lock_guard<std::mutex> lock(mu);
    auto it = state.find(key);
    if (it == state.end()) it = state.emplace(key, no_lean ? LeanChoice() : lean_autotune(F, hbm)).first;
    return it->second;
}

// exported to p2p.cu: the lean geometry and index-tile cap chosen for this factor count and table size (W == 0: general)
bool lean_enabled(int F, long long table_rows) { return lean_choice(F, table_rows).W > 0; }
void lean_geom(int F, long long table_rows, int &W, int &NCH)
{
    const LeanChoice &c = lean_choice(F, table_rows);
    W = c.W;
    NCH = c.NCH;
}
int lean_tile_cap(int F, long long table_rows) { return lean_choice(F, table_rows).tile_cap; }

// which instantiation the last launch_steps call of any thread ran: 0 general, 1 lean, 2 lean user-bucketed; and whether that
// user-bucketed launch ran the staged SGD form (1) or the accumulate-then-sweep one (0)
static std::atomic<int> g_last_step_mode{0}, g_last_step_staged{0};

int launch_steps(StepParams &p, cudaStream_t st, bool keep_status)
{
    // lean: the MF hot path; GEN: any loss but BPR, Adagrad / RMSprop sweeps, FM biases, deterministic accumulation
    StepKernel k = nullptr;
    int tile_cap = kTileDefault, mode = 0, staged = 0;
    bool ub = false;
    if (step_params_lean(p)) {
        const LeanChoice &c = lean_choice(p.F, (long long)p.U + p.I);
        // user-bucketed mode: single-GPU fused steps over uniform batches that update the tables, at least as large as the
        // batch it was timed at (its per-step partition is not amortised by small batches); DRB_UBUCKET=1 takes it at any size
        if (c.ub_W > 0 && p.phases == 3 && p.step_offsets == nullptr && p.apply == 1 && ub_users_for(p.U, p.F, p.batch) > 0 &&
            (p.batch >= kUbTimedBatch || ubucket_switch() == 1)) {
            k = pick_lean_ub(c.ub_W, c.ub_NCH);
            tile_cap = c.tile_cap;
            ub = true;
            mode = 2;
            staged = ub_staged(p, ub_users_for(p.U, p.F, p.batch)) ? 1 : 0;
        } else if (c.W > 0) {
            k = pick_lean_wn(c.W, c.NCH);
            tile_cap = c.tile_cap;
            mode = 1;
        }
    }
    if (k == nullptr) {
        k = pick_kernel(p.F, p.loss != DRB_LOSS_BPR || p.opt > DRB_OPT_ADAM || p.bias != nullptr || p.det != 0);
        tile_cap = kTileDefault;
    }
    DRB_REQUIRE(!p.det || (p.phases == 3 && p.ws.gP64 != nullptr), "deterministic accumulation: single-GPU fused steps with a "
                "workspace from drb_mf_workspace_bytes_det");
    DRB_REQUIRE(k != nullptr, "unsupported factors=%d (row too long for 32 lanes x 8 chunks)", p.F);
    g_last_step_mode = mode;
    g_last_step_staged = staged;
    return launch_kernel(k, p, st, keep_status, tile_cap, ub);
}

int check_nan(void *d_ws, cudaStream_t st, int64_t *nan_step)
{
    WsHeader h;
    DRB_CUDA(cudaMemcpyAsync(&h, d_ws, sizeof(WsHeader), cudaMemcpyDeviceToHost, st));
    DRB_CUDA(cudaStreamSynchronize(st));
    if (h.status == DRB_ERR_NAN_LOSS) {
        if (nan_step) *nan_step = h.nan_step;
        set_error("Loss=Nan or Infinity at step %lld: current settings does not fit the recommender", h.nan_step);
        return DRB_ERR_NAN_LOSS;
    }
    if (nan_step) *nan_step = -1;
    return DRB_OK;
}

}  // namespace drb

using namespace drb;

extern "C" size_t drb_mf_workspace_bytes(int32_t U, int32_t I, int32_t F, int32_t opt)
{
    return carve(nullptr, U, I, F, opt, nullptr);
}

// 1: BPR + SGD/Adam steps at this factor count run the lean instantiation (after its self-check), 2: its user-bucketed mode
// (single-GPU fused steps), 0: the general one.  lanes / chunks (optional) receive the lane geometry of that instantiation.
extern "C" int drb_mf_step_variant(int32_t F, int64_t table_rows, int32_t *lanes, int32_t *chunks)
{
    const drb::LeanChoice &c = drb::lean_choice(F, table_rows);
    const bool bucketed = c.ub_W > 0;
    int W = bucketed ? c.ub_W : c.W, NCH = bucketed ? c.ub_NCH : c.NCH;
    const bool lean = W > 0;
    if (!lean && F > 0) {
        drb::RowGeom g = drb::row_geom(F);
        W = g.width;
        NCH = g.nch;
    }
    if (lanes) *lanes = W;
    if (chunks) *chunks = NCH;
    return bucketed ? 2 : lean ? 1 : 0;
}

// which instantiation the last BPR step launch ran: 0 general, 1 lean, 2 lean user-bucketed (a launch-time choice: the bucketed
// mode also depends on the launch's batch and phases)
extern "C" int drb_mf_last_step_mode(void) { return drb::g_last_step_mode; }

// 1 when that launch ran the user-bucketed mode in its staged SGD form, 0 otherwise (the form depends on the optimiser and the
// bucket width)
extern "C" int drb_mf_last_step_staged(void) { return drb::g_last_step_staged; }

#ifdef DRB_PHASE_TIMERS
// probe build only: the phase timers of the last staged launch (u64 [kPtSteps][kPtMarks][kPtCtas]) into `dst`, and their
// dimensions into dims[3]
extern "C" int drb_phase_timers(void *dst, int32_t *dims)
{
    dims[0] = drb::kPtSteps; dims[1] = drb::kPtMarks; dims[2] = drb::kPtCtas;
    DRB_CUDA(cudaDeviceSynchronize());
    DRB_CUDA(cudaMemcpyFromSymbol(dst, drb::g_phase_t, sizeof(drb::g_phase_t)));
    return DRB_OK;
}
#endif

// the timing half of the on-device selection for `factors`: milliseconds of the timed launch (3 steps of 524 288 triples) of the
// general instantiation and of the best lean candidate, and the index-tile cap in use (runs the selection if it has not run)
extern "C" int drb_mf_step_selfcheck_ms(int32_t F, int64_t table_rows, float *ms_general, float *ms_lean, int32_t *tile_cap)
{
    const drb::LeanChoice &c = drb::lean_choice(F, table_rows);
    if (ms_general) *ms_general = c.ms_general;
    if (ms_lean) *ms_lean = c.ms_lean;
    if (tile_cap) *tile_cap = c.tile_cap;
    return DRB_OK;
}

// host-only: the lane geometry of the lean (lean != 0) or the canonical instantiation for `factors`, and the tile size the
// launcher picks for `per_cta` triples per CTA and step (no device needed)
extern "C" int drb_mf_step_geometry(int32_t F, int32_t lean, int32_t *lanes, int32_t *chunks, int64_t per_cta, int32_t *tile)
{
    int W = 0, NCH = 0;
    if (lean) {
        drb::lean_default_geom(F, W, NCH);
    } else if (F > 0) {
        drb::RowGeom g = drb::row_geom(F);
        W = g.width;
        NCH = g.nch;
    }
    if (lanes) *lanes = W;
    if (chunks) *chunks = NCH;
    if (tile) *tile = drb::pick_tile(per_cta);
    return W > 0 ? DRB_OK : DRB_ERR_INVALID;
}

extern "C" int drb_mf_workspace_init(void *d_ws, int32_t U, int32_t I, int32_t F, int32_t opt, void *stream)
{
    DRB_REQUIRE(d_ws != nullptr && U > 0 && I > 0 && F > 0, "workspace_init: bad arguments");
    size_t bytes = carve(nullptr, U, I, F, opt, nullptr);
    DRB_CUDA(cudaMemsetAsync(d_ws, 0, bytes, (cudaStream_t)stream));
    return DRB_OK;
}

namespace drb {
int fill_params(StepParams &p, float *P, float *Q, void *d_ws, int U, int I, int F, const int32_t *bu, const int32_t *bi,
                const int32_t *bj, long long n, long long batch, long long first, long long nsteps, const drb_hyper *h,
                long long adam_step0, double *d_step_loss, int apply, float *d_bias, int det)
{
    DRB_REQUIRE(P && Q && d_ws && bu && bi && bj && h && d_step_loss, "null pointer argument");
    DRB_REQUIRE(U > 0 && I > 0 && F > 0 && batch > 0 && n >= 0 && first >= 0 && nsteps >= 0, "bad sizes");
    DRB_REQUIRE(h->opt >= DRB_OPT_SGD && h->opt <= DRB_OPT_RMSPROP, "unknown optimizer id %d", h->opt);
    DRB_REQUIRE(h->loss >= DRB_LOSS_BPR && h->loss <= DRB_LOSS_SL, "unknown loss id %d", h->loss);
    DRB_REQUIRE((first + nsteps - 1) * batch < n || nsteps == 0 || n == 0, "steps [%lld,%lld) exceed %lld triples", first,
                first + nsteps, n);
    p = one_step(h, U, I, F, bu, bi, bj, batch, adam_step0);
    p.n = n; p.first_step = first; p.n_steps = nsteps;
    p.P = P; p.Q = Q;
    carve(d_ws, U, I, F, h->opt, &p.ws, d_bias != nullptr, det);
    p.det = det;
    p.step_loss = d_step_loss;
    p.apply = apply;
    p.bias = d_bias;
    return DRB_OK;
}
}  // namespace drb

extern "C" int drb_mf_bpr_train_steps(float *d_P, float *d_Q, void *d_ws, int32_t U, int32_t I, int32_t F,
                                      const int32_t *d_bu, const int32_t *d_bi, const int32_t *d_bj, int64_t n,
                                      int64_t batch, int64_t first_step, int64_t n_steps, const drb_hyper *hyper,
                                      int64_t adam_step0, double *d_step_loss, int32_t sync_and_check,
                                      int64_t *nan_step, void *stream)
{
    StepParams p;
    int rc = fill_params(p, d_P, d_Q, d_ws, U, I, F, d_bu, d_bi, d_bj, n, batch, first_step, n_steps, hyper, adam_step0,
                         d_step_loss, 1);
    if (rc != DRB_OK) return rc;
    if (n_steps == 0) return DRB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    rc = launch_steps(p, st);
    if (rc != DRB_OK) return rc;
    if (sync_and_check) return check_nan(d_ws, st, nan_step);
    return DRB_OK;
}

// Deterministic accumulation (opt-in): the same steps with every cross-thread sum taken in fixed point, so that two runs --
// and any two orders of the atomics -- give bitwise identical tables and losses.  Workspace: drb_mf_workspace_bytes_det.
extern "C" size_t drb_mf_workspace_bytes_det(int32_t U, int32_t I, int32_t F, int32_t opt)
{
    return carve(nullptr, U, I, F, opt, nullptr, 0, 1);
}

extern "C" int drb_mf_bpr_train_steps_det(float *d_P, float *d_Q, void *d_ws, int32_t U, int32_t I, int32_t F,
                                          const int32_t *d_bu, const int32_t *d_bi, const int32_t *d_bj, int64_t n,
                                          int64_t batch, int64_t first_step, int64_t n_steps, const drb_hyper *hyper,
                                          int64_t adam_step0, double *d_step_loss, int32_t sync_and_check, int64_t *nan_step,
                                          void *stream)
{
    StepParams p;
    int rc = fill_params(p, d_P, d_Q, d_ws, U, I, F, d_bu, d_bi, d_bj, n, batch, first_step, n_steps, hyper, adam_step0,
                         d_step_loss, 1, nullptr, 1);
    if (rc != DRB_OK) return rc;
    if (n_steps == 0) return DRB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    rc = launch_steps(p, st);
    if (rc != DRB_OK) return rc;
    if (sync_and_check) return check_nan(d_ws, st, nan_step);
    return DRB_OK;
}

extern "C" int drb_mf_bpr_train_steps_fused_neg(float *d_P, float *d_Q, void *d_ws, int32_t U, int32_t I, int32_t F,
                                                const int32_t *d_bu, const int32_t *d_bi, const int64_t *d_row_ptr,
                                                const int32_t *d_col, uint64_t seed, int32_t *d_neg_out, int64_t n,
                                                int64_t batch, int64_t first_step, int64_t n_steps, const drb_hyper *hyper,
                                                int64_t adam_step0, double *d_step_loss, int32_t sync_and_check,
                                                int64_t *nan_step, void *stream)
{
    DRB_REQUIRE(d_row_ptr && d_col, "train_steps_fused_neg: the user->item CSR is required");
    DRB_REQUIRE(hyper && hyper->loss < DRB_LOSS_CL, "train_steps_fused_neg: pair-wise losses only");
    StepParams p;
    // the negative plane is unused in this mode (bi stands in so that the TMA staging code stays uniform)
    int rc = fill_params(p, d_P, d_Q, d_ws, U, I, F, d_bu, d_bi, d_bi, n, batch, first_step, n_steps, hyper, adam_step0,
                         d_step_loss, 1);
    if (rc != DRB_OK) return rc;
    if (n_steps == 0) return DRB_OK;
    p.neg_row_ptr = d_row_ptr;
    p.neg_col = d_col;
    p.neg_out = d_neg_out;
    p.neg_seed = seed;
    p.dense_hint = 1;   // phase 2 must not re-derive negatives: dense sweep only
    cudaStream_t st = (cudaStream_t)stream;
    rc = launch_steps(p, st);
    if (rc != DRB_OK) return rc;
    if (sync_and_check) return check_nan(d_ws, st, nan_step);
    return DRB_OK;
}

extern "C" int drb_mf_bpr_loss(const float *d_P, const float *d_Q, void *d_ws, int32_t U, int32_t I, int32_t F,
                               const int32_t *d_bu, const int32_t *d_bi, const int32_t *d_bj, int64_t batch,
                               const drb_hyper *hyper, double *d_loss, void *stream)
{
    StepParams p;
    int rc = fill_params(p, (float *)d_P, (float *)d_Q, d_ws, U, I, F, d_bu, d_bi, d_bj, batch, batch, 0, 1, hyper, 0,
                         d_loss, 0);
    if (rc != DRB_OK) return rc;
    return launch_steps(p, (cudaStream_t)stream);
}

// ---- FM (daisy/model/FMRecommender.py:61-97): the MF step with first-order terms; d_bias = [u_bias (U), i_bias (I), bias_]
extern "C" size_t drb_fm_workspace_bytes(int32_t U, int32_t I, int32_t F, int32_t opt)
{
    return carve(nullptr, U, I, F, opt, nullptr, 1);
}

extern "C" int drb_fm_workspace_init(void *d_ws, int32_t U, int32_t I, int32_t F, int32_t opt, void *stream)
{
    DRB_REQUIRE(d_ws != nullptr && U > 0 && I > 0 && F > 0, "fm_workspace_init: bad arguments");
    DRB_CUDA(cudaMemsetAsync(d_ws, 0, carve(nullptr, U, I, F, opt, nullptr, 1), (cudaStream_t)stream));
    return DRB_OK;
}

extern "C" int drb_fm_train_steps(float *d_P, float *d_Q, float *d_bias, void *d_ws, int32_t U, int32_t I, int32_t F,
                                  const int32_t *d_bu, const int32_t *d_bi, const int32_t *d_bj, int64_t n, int64_t batch,
                                  int64_t first_step, int64_t n_steps, const drb_hyper *hyper, int64_t adam_step0,
                                  int32_t apply, double *d_step_loss, int32_t sync_and_check, int64_t *nan_step, void *stream)
{
    DRB_REQUIRE(d_bias != nullptr, "fm_train_steps: the bias vector is required");
    StepParams p;
    int rc = fill_params(p, d_P, d_Q, d_ws, U, I, F, d_bu, d_bi, d_bj, n, batch, first_step, n_steps, hyper, adam_step0,
                         d_step_loss, apply ? 1 : 0, d_bias);
    if (rc != DRB_OK) return rc;
    if (n_steps == 0) return DRB_OK;
    DRB_REQUIRE(apply || n_steps == 1, "fm_train_steps: apply=0 evaluates the loss of ONE batch");
    cudaStream_t st = (cudaStream_t)stream;
    rc = launch_steps(p, st);
    if (rc != DRB_OK) return rc;
    if (sync_and_check) return check_nan(d_ws, st, nan_step);
    return DRB_OK;
}

extern "C" int drb_mf_bpr_train_step_host(float *d_P, float *d_Q, void *d_ws, int32_t U, int32_t I, int32_t F,
                                          const int32_t *h_bu, const int32_t *h_bi, const int32_t *h_bj, int64_t batch,
                                          const drb_hyper *hyper, int64_t adam_step0, int32_t *d_stage, double *h_loss,
                                          void *stream)
{
    DRB_REQUIRE(h_bu && h_bi && h_bj && d_stage && h_loss && batch > 0, "train_step_host: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    size_t stride = (size_t)((batch + 3) / 4 * 4);  // keep each array 16-byte aligned for the TMA path
    size_t bytes = sizeof(int32_t) * (size_t)batch;
    DRB_CUDA(cudaMemcpyAsync(d_stage, h_bu, bytes, cudaMemcpyHostToDevice, st));
    DRB_CUDA(cudaMemcpyAsync(d_stage + stride, h_bi, bytes, cudaMemcpyHostToDevice, st));
    DRB_CUDA(cudaMemcpyAsync(d_stage + 2 * stride, h_bj, bytes, cudaMemcpyHostToDevice, st));
    double *d_loss = (double *)(d_stage + 3 * stride);
    StepParams p;
    int rc = fill_params(p, d_P, d_Q, d_ws, U, I, F, d_stage, d_stage + stride, d_stage + 2 * stride, batch, batch, 0, 1,
                         hyper, adam_step0, d_loss, 1);
    if (rc != DRB_OK) return rc;
    rc = launch_steps(p, st);
    if (rc != DRB_OK) return rc;
    DRB_CUDA(cudaMemcpyAsync(h_loss, d_loss, sizeof(double), cudaMemcpyDeviceToHost, st));
    int64_t nan_step = -1;
    return check_nan(d_ws, st, &nan_step);
}

// Pipelined end-to-end steps from HOST index planes: the H2D copy of step s+1 (copy stream) overlaps the
// kernel of step s (compute stream); every step's loss is read back to the host asynchronously.
extern "C" int drb_mf_bpr_train_steps_host(float *d_P, float *d_Q, void *d_ws, int32_t U, int32_t I, int32_t F,
                                           const int32_t *h_bu, const int32_t *h_bi, const int32_t *h_bj, int64_t n,
                                           int64_t batch, int64_t n_steps, const drb_hyper *hyper, int64_t adam_step0,
                                           int32_t *d_stage, double *d_loss, double *h_loss, int64_t *nan_step,
                                           void *stream)
{
    DRB_REQUIRE(h_bu && h_bi && h_bj && d_stage && d_loss && h_loss && batch > 0 && n_steps >= 0 && n >= 0,
                "train_steps_host: bad arguments");
    DRB_REQUIRE(n_steps == 0 || (n_steps - 1) * batch < n, "train_steps_host: %lld steps exceed %lld triples",
                (long long)n_steps, (long long)n);
    if (n_steps == 0) return DRB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    static thread_local cudaStream_t copy_st = nullptr;
    if (!copy_st) DRB_CUDA(cudaStreamCreateWithFlags(&copy_st, cudaStreamNonBlocking));
    cudaEvent_t ready[2], freed[2], start;
    for (int k = 0; k < 2; ++k) {
        DRB_CUDA(cudaEventCreateWithFlags(&ready[k], cudaEventDisableTiming));
        DRB_CUDA(cudaEventCreateWithFlags(&freed[k], cudaEventDisableTiming));
    }
    DRB_CUDA(cudaEventCreateWithFlags(&start, cudaEventDisableTiming));
    const size_t stride = (size_t)((batch + 3) / 4 * 4);
    DRB_CUDA(cudaMemsetAsync(d_ws, 0, sizeof(WsHeader), st));   // clear a stale NaN flag once; sticky afterwards
    DRB_CUDA(cudaEventRecord(start, st));
    DRB_CUDA(cudaStreamWaitEvent(copy_st, start, 0));            // staging slots may still be in use upstream
    int rc = DRB_OK;
    for (int64_t s = 0; s < n_steps && rc == DRB_OK; ++s) {
        const int slot = (int)(s & 1);
        int32_t *sb = d_stage + (size_t)slot * 3 * stride;
        const int64_t base = s * batch, nb = (n - base < batch) ? n - base : batch;
        const size_t bytes = sizeof(int32_t) * (size_t)nb;
        if (s >= 2) DRB_CUDA(cudaStreamWaitEvent(copy_st, freed[slot], 0));
        DRB_CUDA(cudaMemcpyAsync(sb, h_bu + base, bytes, cudaMemcpyHostToDevice, copy_st));
        DRB_CUDA(cudaMemcpyAsync(sb + stride, h_bi + base, bytes, cudaMemcpyHostToDevice, copy_st));
        DRB_CUDA(cudaMemcpyAsync(sb + 2 * stride, h_bj + base, bytes, cudaMemcpyHostToDevice, copy_st));
        DRB_CUDA(cudaEventRecord(ready[slot], copy_st));
        DRB_CUDA(cudaStreamWaitEvent(st, ready[slot], 0));
        StepParams p;
        rc = fill_params(p, d_P, d_Q, d_ws, U, I, F, sb, sb + stride, sb + 2 * stride, nb, nb, 0, 1, hyper, adam_step0 + s,
                         d_loss + s, 1);
        if (rc == DRB_OK) rc = launch_steps(p, st, /*keep_status=*/true);
        if (rc != DRB_OK) break;
        DRB_CUDA(cudaEventRecord(freed[slot], st));
        DRB_CUDA(cudaMemcpyAsync(h_loss + s, d_loss + s, sizeof(double), cudaMemcpyDeviceToHost, st));
    }
    int rc2 = (rc == DRB_OK) ? check_nan(d_ws, st, nan_step) : rc;
    cudaStreamSynchronize(copy_st);
    for (int k = 0; k < 2; ++k) {
        cudaEventDestroy(ready[k]);
        cudaEventDestroy(freed[k]);
    }
    cudaEventDestroy(start);
    return rc2;
}

extern "C" int drb_gather_triples(const int32_t *d_triples, const int64_t *d_perm, int64_t n, int32_t *d_bu,
                                  int32_t *d_bi, int32_t *d_bj, void *stream)
{
    DRB_REQUIRE(d_triples && d_bu && d_bi && d_bj && n >= 0, "gather_triples: bad arguments");
    if (n == 0) return DRB_OK;
    gather_triples_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(d_triples, d_perm, n, d_bu, d_bi, d_bj);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}

extern "C" int drb_mf_workspace_layout(int32_t U, int32_t I, int32_t F, int32_t opt, int64_t *out8)
{
    DRB_REQUIRE(out8 && U > 0 && I > 0 && F > 0, "workspace_layout: bad arguments");
    Workspace w;
    carve((void *)(uintptr_t)256, U, I, F, opt, &w);   // fake non-null base: pointers become offsets + 256
    auto off = [](const void *p) { return (int64_t)((uintptr_t)p - 256); };
    out8[0] = off(&w.hdr->acc[0][0]);  out8[1] = 8 * sizeof(double);
    out8[2] = off(w.gQ);               out8[3] = (int64_t)sizeof(float) * I * F;
    out8[4] = off(w.cntI);             out8[5] = (int64_t)sizeof(unsigned long long) * I;
    out8[6] = off(w.gP);               out8[7] = off(w.cntU);
    return DRB_OK;
}

extern "C" int drb_mf_bpr_phase(float *d_P, float *d_Q, void *d_ws, int32_t U, int32_t I, int32_t F, const int32_t *d_bu,
                                const int32_t *d_bi, const int32_t *d_bj, int64_t begin, int64_t count, int32_t phase,
                                const drb_hyper *hyper, int64_t adam_step0, double *d_loss, void *stream)
{
    DRB_REQUIRE(phase == 1 || phase == 2, "mf_bpr_phase: phase must be 1 or 2");
    DRB_REQUIRE(begin >= 0 && count >= 0, "mf_bpr_phase: bad range");
    DRB_REQUIRE(hyper && hyper->loss < DRB_LOSS_CL, "mf_bpr_phase: the sharded step covers the pair-wise losses only");
    StepParams p;
    // count may be 0 on a rank (its users have no triple in this global batch): phases still run (loss, sweep)
    int rc = fill_params(p, d_P, d_Q, d_ws, U, I, F, d_bu + begin, d_bi + begin, d_bj + begin, count, count > 0 ? count : 1,
                         0, 1, hyper, adam_step0, d_loss, 1);
    if (rc != DRB_OK) return rc;
    p.phases = phase;
    p.dense_hint = 1;
    return launch_steps(p, (cudaStream_t)stream);
}
