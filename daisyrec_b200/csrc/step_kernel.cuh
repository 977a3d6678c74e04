// step_kernel.cuh -- device code of the BPR step kernel (see the header of mf_bpr.cu for the algorithm), shared by the
// single-GPU persistent kernel (mf_bpr.cu) and the peer-exchange multi-GPU kernel (p2p.cu).  The body is a template over an
// EXCHANGE policy: NoExchange compiles to exactly the single-GPU kernel; P2PExchange (p2p.cu) redirects the item-side
// accumulators into a peer-visible buffer, rendezvouses with the other ranks between the phases and replaces the item half of
// the phase-2 sweep with a reduce-update-broadcast of this rank's item slice over NVLink.
#pragma once
#include <math.h>
#include <stdlib.h>

#include "step.cuh"

namespace drb {

constexpr int kThreads = 256;
constexpr int kTileMax = 1024;  // triples per staged index tile

constexpr int kTileDefault = 512;
constexpr int kUbMaxRows = 512;   // users per bucket of the user-bucketed mode at most (its per-tile sort keys)

// Tile size for `per_cta` triples per CTA and step: the fewest equal tiles of at most `cap` triples (a multiple of 16), so every
// CTA walks the same number of full tiles (cap 512: 3 543 per CTA -> 7 tiles of 512; cap 1 024 -> 4 tiles of 896).
inline int pick_tile(long long per_cta, int cap = kTileDefault)
{
    static const int forced = [] {
        const char *e = getenv("DRB_TILE_CAP");   // developer switch
        int c = e ? atoi(e) : 0;
        return (c >= 16 && c <= kTileMax) ? c / 16 * 16 : 0;
    }();
    if (forced) cap = forced;
    if (cap > kTileMax) cap = kTileMax;
    if (cap < 16) cap = 16;
    if (per_cta < 16) return 16;
    const long long k = (per_cta + cap - 1) / cap;
    long long tile = ((per_cta + k - 1) / k + 15) / 16 * 16;
    return (int)(tile > cap ? cap : tile);
}
#ifndef DRB_MINB
#define DRB_MINB 2             // resident CTAs per SM the register allocator must allow
#endif
#ifndef DRB_UNR
#define DRB_UNR 2              // triples in flight per lane group (memory-level parallelism)
#endif

// Phase timers of the staged user-bucketed form, compiled in only by the probe build (-DDRB_PHASE_TIMERS,
// scripts/probe_mf_phases.py --timers): thread 0 of every CTA writes %globaltimer at each phase boundary of the first
// kPtSteps steps of a launch into g_phase_t[step][mark][cta]; drb_phase_timers (mf_bpr.cu) copies it to the host.
#ifdef DRB_PHASE_TIMERS
constexpr int kPtSteps = 96, kPtMarks = 12, kPtCtas = 512;
__device__ unsigned long long g_phase_t[kPtSteps][kPtMarks][kPtCtas];
__device__ __forceinline__ void phase_mark(long long s, int m)
{
    if (threadIdx.x == 0 && s < kPtSteps && blockIdx.x < kPtCtas) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)::"memory");
        g_phase_t[s][m][blockIdx.x] = t;
    }
}
#else
__device__ __forceinline__ void phase_mark(long long, int) {}
#endif

// ------------------------------------------------------------------ device pieces
// deterministic mode: contribution -> 2^40 fixed point (|sum| < 2^23 = 8.4e6, resolution 9e-13).  The step's scalar sums, each
// lane's share of one triple rounded on its own (that share depends on the row geometry alone, so the integer totals do not
// depend on how triples map to threads: tile size, grid, SM count): the loss -> 2^24 (|sum| < 2^39 = 5.5e11, resolution 6e-8),
// the l1 and squared-norm sums of the batch rows -> 2^32 (|sum| < 2^31 = 2.1e9, resolution 2.3e-10: the batch norms, and
// through them the reg_2 term, stay as close to fp64 as the fp32 partials were).  No range bounds what a diverging run reaches
// (SL's (x - y)^2 and HL's margin are unbounded), so every value and every integer addition is checked: a non-finite value,
// one of 2^62 units or more, or an addition that overflows int64 makes the step report a non-finite loss (DRB_ERR_NAN_LOSS)
// before phase 2 applies it.
constexpr double kDetScale = 1099511627776.0, kDetAccScale = 16777216.0, kDetNormScale = 4294967296.0;
constexpr double kDetValueMax = 4611686018427387904.0;   // 2^62

__device__ __forceinline__ float sgnf(float x) { return (float)((x > 0.f) - (x < 0.f)); }

struct Norms {
    float inv_u, inv_i, inv_j;  // 1/||.||_F, 0 when the norm is 0 (zero subgradient)
};

struct AdamCoef {
    float step_size, bc2_sqrt;
};

// Gradient of one element of a touched row: its accumulated part g plus the regulariser, count x f(theta), for the row's two
// roles (ca / cb occurrences, ia / ib the inverse batch norms; user rows: cb = 0).  The dense sweep and the bucketed SGD user
// update (bpr_steps_body) both take it from here, so they compile the same fp32 expression.
__device__ __forceinline__ float reg_grad(float x, float g, float ca, float ia, float cb, float ib, const StepParams &p)
{
    const float sg = p.reg1 * sgnf(x);
    return g + (ca * (sg + p.reg2 * x * ia) + cb * (sg + p.reg2 * x * ib));
}

// The regulariser of reg_grad for ONE occurrence of a row (ia: the inverse batch norm of its role): the bucketed SGD step adds
// it to each item gradient contribution in phase 1, the order in which autograd sums the reference's loss
__device__ __forceinline__ float reg_term(float x, float ia, const StepParams &p)
{
    return p.reg1 * sgnf(x) + p.reg2 * x * ia;
}

// ||row||^2 and ||row||_1 of a user row of CH 4-float chunks, one chunk per lane: the CH lanes of a row are consecutive and CH
// divides 32, so xor-shuffles within them finish both sums (every lane of the warp must take part)
template <int CH>
__device__ __forceinline__ float2 row_norms(float4 v)
{
    float s2 = 0.f, l1 = 0.f;
    s2 = fmaf(v.x, v.x, s2); s2 = fmaf(v.y, v.y, s2); s2 = fmaf(v.z, v.z, s2); s2 = fmaf(v.w, v.w, s2);
    l1 = fabsf(v.x) + fabsf(v.y) + fabsf(v.z) + fabsf(v.w);
#pragma unroll
    for (int off = 1; off < CH; off <<= 1) {
        s2 += __shfl_xor_sync(0xffffffffu, s2, off);
        l1 += __shfl_xor_sync(0xffffffffu, l1, off);
    }
    return make_float2(s2, l1);
}

// Apply the accumulated gradient of ONE table row (all W lanes of the group cooperate).
// cnt_a / cnt_b: occurrences weighted by inv_a / inv_b (user rows: cnt_b = 0).
template <int VEC, int W, int NCH, int OPT>
__device__ __forceinline__ void apply_row(float *theta_row, float *g_row, float *m_row, float *v_row, int gl,
                                          int chunks, float cnt_a, float inv_a, float cnt_b, float inv_b,
                                          const StepParams &p, const AdamCoef &ac, bool touched)
{
#pragma unroll
    for (int ch = 0; ch < NCH; ++ch) {
        int c = gl + ch * W;
        if (c >= chunks) continue;
        float *tp = theta_row + c * VEC;
        Vec<VEC> th = ld_row<VEC>(tp);
        Vec<VEC> g;
        if (touched) {
            g = ld_row<VEC>(g_row + c * VEC);
            Vec<VEC> z;
#pragma unroll
            for (int e = 0; e < VEC; ++e) z.v[e] = 0.f;
            st_row<VEC>(g_row + c * VEC, z);
        } else {
#pragma unroll
            for (int e = 0; e < VEC; ++e) g.v[e] = 0.f;
        }
#pragma unroll
        for (int e = 0; e < VEC; ++e) {
            float t = th.v[e];
            float gg = g.v[e];
            if (touched) {
                float sg = p.reg1 * sgnf(t);
                gg += cnt_a * (sg + p.reg2 * t * inv_a) + cnt_b * (sg + p.reg2 * t * inv_b);
            }
            g.v[e] = gg;
        }
        if constexpr (OPT == DRB_OPT_SGD) {
#pragma unroll
            for (int e = 0; e < VEC; ++e) th.v[e] = th.v[e] - p.lr * g.v[e];
        } else {
            Vec<VEC> m = ld_row<VEC>(m_row + c * VEC), v = ld_row<VEC>(v_row + c * VEC);
#pragma unroll
            for (int e = 0; e < VEC; ++e) {
                float gk = g.v[e];
                m.v[e] = m.v[e] + (gk - m.v[e]) * (1.f - p.beta1);
                v.v[e] = v.v[e] * p.beta2 + (1.f - p.beta2) * gk * gk;
                float denom = sqrtf(v.v[e]) / ac.bc2_sqrt + p.eps;
                th.v[e] = th.v[e] - ac.step_size * (m.v[e] / denom);
            }
            st_row<VEC>(m_row + c * VEC, m);
            st_row<VEC>(v_row + c * VEC, v);
        }
        st_row<VEC>(tp, th);
    }
}

// Dense phase-2 sweep: lane groups walk ALL rows of P then Q, R rows in flight each.  Counter, theta
// and gradient accumulator of the R rows are loaded unconditionally and up front (one memory round
// trip instead of three dependent ones); an untouched SGD row has cnt == 0 and g == 0, so nothing is
// written for it.  Adam moves every row (dense optimiser semantics of the reference).  Adagrad / RMSprop
// (AbstractRecommender.py:57-60, torch defaults) keep ONE state row in the m slot: Adagrad leaves an untouched row
// alone (g = 0 adds nothing), RMSprop's running square of an untouched row still decays by alpha.
// DET (deterministic mode): the gradient is read from the fixed-point sums and assembled with the regulariser in fp64, rounded
// to fp32 once, and the SGD step rounds lr * g before the subtraction -- the fp64-accumulating oracle's arithmetic, so that the
// result does not depend on how the compiler contracts the fp32 expression.
// USERS_ONLY: the user rows alone (peer exchange: item rows have an owner rank).
template <int VEC, int W, int NCH, int OPT, bool USERS_ONLY = false, bool DET = false>
__device__ __forceinline__ void dense_sweep(const StepParams &p, const Norms &nm, const AdamCoef &ac, int gl, int group,
                                            int groups_per_cta, int chunks)
{
    constexpr int R = (OPT == DRB_OPT_SGD) ? ((NCH * VEC <= 4) ? 4 : 2) : ((NCH * VEC <= 4) ? 2 : 1);
    const long long rows = USERS_ONLY ? (long long)p.U : (long long)p.U + p.I;
    const long long tg = (long long)gridDim.x * groups_per_cta;
    const int F = p.F;
    for (long long r0 = (long long)blockIdx.x * groups_per_cta + group; r0 < rows; r0 += tg * R) {
        float *th_p[R], *g_p[R], *m_p[R], *v_p[R];
        long long *g64_p[R];
        unsigned long long cnt[R];
        bool act[R], is_user[R];
        Row<VEC, W, NCH> th[R], g[R], m[R], v[R];
#pragma unroll
        for (int k = 0; k < R; ++k) {
            long long r = r0 + (long long)k * tg;
            act[k] = r < rows;
            is_user[k] = r < p.U;
            long long it = is_user[k] ? r : r - p.U;
            size_t o = (size_t)(act[k] ? it : 0) * F;
            th_p[k] = (is_user[k] ? p.P : p.Q) + o;
            g_p[k] = (is_user[k] ? p.ws.gP : p.ws.gQ) + o;
            if constexpr (DET) g64_p[k] = (is_user[k] ? p.ws.gP64 : p.ws.gQ64) + o;
            cnt[k] = 0;
            if (act[k]) cnt[k] = is_user[k] ? (unsigned long long)__ldcg(p.ws.cntU + it) : __ldcg(p.ws.cntI + it);
            th[k] = load_row<VEC, W, NCH>(th_p[k], gl, chunks, act[k]);
            g[k] = load_row<VEC, W, NCH>(g_p[k], gl, chunks, act[k]);
            if constexpr (OPT != DRB_OPT_SGD) {
                m_p[k] = (is_user[k] ? p.ws.mP : p.ws.mQ) + o;
                m[k] = load_row<VEC, W, NCH>(m_p[k], gl, chunks, act[k]);
            }
            if constexpr (OPT == DRB_OPT_ADAM) {
                v_p[k] = (is_user[k] ? p.ws.vP : p.ws.vQ) + o;
                v[k] = load_row<VEC, W, NCH>(v_p[k], gl, chunks, act[k]);
            }
        }
#pragma unroll
        for (int k = 0; k < R; ++k) {
            const bool touched = cnt[k] != 0;
            if (!act[k] || ((OPT == DRB_OPT_SGD || OPT == DRB_OPT_ADAGRAD) && !touched && !p.dense_grad)) continue;
            const float ca = (float)(unsigned)(cnt[k] & 0xffffffffull), cb = p.neg_mult * (float)(unsigned)(cnt[k] >> 32);
            const float ia = is_user[k] ? nm.inv_u : nm.inv_i, ib = nm.inv_j;
#pragma unroll
            for (int ch = 0; ch < NCH; ++ch) {
                int c = gl + ch * W;
                if (c >= chunks) continue;
                Vec<VEC> &t = th[k].c[ch];
#pragma unroll
                for (int e = 0; e < VEC; ++e) {
                    float x = t.v[e], gg;
                    if constexpr (DET) {
                        long long *fx_p = g64_p[k] + c * VEC + e;
                        const long long fx = __ldcg(fx_p);
                        double gd = (double)p.gscale * ((double)fx / kDetScale);
                        if (touched) {
                            const double sg = (double)(p.reg1 * sgnf(x));
                            gd += (double)ca * (sg + (double)__fmul_rn(__fmul_rn(p.reg2, x), ia)) +
                                  (double)cb * (sg + (double)__fmul_rn(__fmul_rn(p.reg2, x), ib));
                        }
                        if (fx != 0) __stcg(fx_p, 0ll);
                        gg = (float)gd;
                    } else {
                        gg = p.gscale * g[k].c[ch].v[e];
                        if (touched) gg = reg_grad(x, gg, ca, ia, cb, ib, p);
                    }
                    if constexpr (OPT == DRB_OPT_SGD) {
                        t.v[e] = DET ? __fsub_rn(x, __fmul_rn(p.lr, gg)) : x - p.lr * gg;
                    } else if constexpr (OPT == DRB_OPT_ADAGRAD) {   // sum += g^2; theta -= lr g / (sqrt(sum) + 1e-10)
                        float ss = m[k].c[ch].v[e] + gg * gg;
                        t.v[e] = x - p.lr * (gg / (sqrtf(ss) + 1e-10f));
                        m[k].c[ch].v[e] = ss;
                    } else if constexpr (OPT == DRB_OPT_RMSPROP) {   // sq = .99 sq + .01 g^2; theta -= lr g / (sqrt(sq) + 1e-8)
                        float sq = m[k].c[ch].v[e] * 0.99f + (1.f - 0.99f) * gg * gg;
                        t.v[e] = x - p.lr * (gg / (sqrtf(sq) + 1e-8f));
                        m[k].c[ch].v[e] = sq;
                    } else {
                        float mm = m[k].c[ch].v[e], vv = v[k].c[ch].v[e];
                        mm = mm + (gg - mm) * (1.f - p.beta1);
                        vv = vv * p.beta2 + (1.f - p.beta2) * gg * gg;
                        float denom = sqrtf(vv) / ac.bc2_sqrt + p.eps;
                        t.v[e] = x - ac.step_size * (mm / denom);
                        m[k].c[ch].v[e] = mm;
                        v[k].c[ch].v[e] = vv;
                    }
                }
                st_row<VEC>(th_p[k] + c * VEC, t);
                if constexpr (OPT != DRB_OPT_SGD) st_row<VEC>(m_p[k] + c * VEC, m[k].c[ch]);
                if constexpr (OPT == DRB_OPT_ADAM) st_row<VEC>(v_p[k] + c * VEC, v[k].c[ch]);
                if (touched) {
                    Vec<VEC> z;
#pragma unroll
                    for (int e = 0; e < VEC; ++e) z.v[e] = 0.f;
                    st_row<VEC>(g_p[k] + c * VEC, z);
                }
            }
            if (touched && gl == 0 && !p.keep_counts) {
                long long r = r0 + (long long)k * tg;
                if (is_user[k]) p.ws.cntU[r] = 0u; else p.ws.cntI[r - p.U] = 0ull;
            }
        }
    }
}

// Fresh uniform negative for (user u, global triple index gt, step): a Philox word scaled to [0, n_comp) by multiply-high,
// then the k-th item missing from the user's sorted row: item = k + #{s : col[s] - s <= k} (one binary search).
__device__ __forceinline__ int draw_negative(const StepParams &p, int u, unsigned long long gt, unsigned long long step)
{
    const long long rb = p.neg_row_ptr[u], re = p.neg_row_ptr[u + 1];
    const unsigned n_comp = (unsigned)((long long)p.I - (re - rb));
    uint32_t c[4] = {(uint32_t)gt, (uint32_t)(gt >> 32), (uint32_t)step, (uint32_t)(step >> 32)};
    philox4x32(c, (uint32_t)p.neg_seed, (uint32_t)(p.neg_seed >> 32));
    const int k = (int)__umulhi(c[0], n_comp);
    long long lo = 0, hi = re - rb;
    while (lo < hi) {
        long long mid = (lo + hi) >> 1;
        if ((long long)__ldg(p.neg_col + rb + mid) - mid <= (long long)k) lo = mid + 1; else hi = mid;
    }
    const int item = k + (int)lo;
    return item < p.I ? item : p.I - 1;   // only reachable for a user who interacted with every item (rejected by the host)
}

template <bool LEAN> struct RowOffset { typedef size_t type; };
template <> struct RowOffset<true> { typedef unsigned type; };

// deterministic mode: a + b in int64; ok becomes false when the sum overflows
__device__ __forceinline__ long long det_add(long long a, long long b, bool &ok)
{
    const long long s = (long long)((unsigned long long)a + (unsigned long long)b);
    ok = ok && ((a ^ s) & (b ^ s)) >= 0;
    return s;
}

// deterministic mode: v in `scale` fixed point; ok becomes false for a non-finite value or one of 2^62 units or more
__device__ __forceinline__ long long det_fix(float v, double scale, bool &ok)
{
    const double s = (double)v * scale;
    if (!(fabs(s) < kDetValueMax)) { ok = false; return 0; }
    return __double2ll_rn(s);
}

// deterministic mode: add one contribution to a table element's fixed-point sum; the returned old value shows an overflow of
// the sum.  A sum whose final value leaves the int64 range crosses it in every order of the additions, so it is always seen.
__device__ __forceinline__ void det_red(long long *p, float v, bool &ok)
{
    const long long x = det_fix(v, kDetScale, ok);
    if (x == 0) return;
    const long long old = (long long)atomicAdd(reinterpret_cast<unsigned long long *>(p), (unsigned long long)x);
    det_add(old, x, ok);
}

// Exchange policy of the single-GPU kernel: nothing to exchange (every hook is a compile-time no-op).
struct NoExchange {
    static constexpr bool kActive = false;
    __device__ __forceinline__ void begin_step(StepParams &, long long, double *&) {}
    __device__ __forceinline__ bool after_phase1(const StepParams &, long long, double *&, unsigned long long &) { return true; }
    template <int VEC, int W, int NCH>
    __device__ __forceinline__ void item_slice(const StepParams &, long long, const Norms &, const AdamCoef &, int, int, int,
                                               int, unsigned long long &) {}
    __device__ __forceinline__ bool end_step(const StepParams &, long long, unsigned long long &) { return true; }
};

// LEAN: the MF hot instantiation (launch_steps picks it when the parameters allow): BPR, no ego / norm tables (LightGCN),
// no in-kernel negative draw, and 32-bit element offsets into the tables (rows * F < 2^32) -- the same arithmetic on the same
// operands in the same order as the general body, with ~1/3 fewer instructions per triple.
//
// UBK (user-bucketed, lean single-GPU fused steps only): every step first partitions its triples by user bucket into scratch
// records (histogram, grid barrier, scan + reservation, scatter, grid barrier); phase 1 then has CTAs claim whole buckets, sort
// each tile of the bucket by user, sum the user gradient of each run of a user in registers, add the run sums and the counts of
// the bucket in shared memory and write each touched gP row and cntU entry once with plain stores, instead of one RED per
// occurrence into the (L2-missing) user accumulators.  Item side, loss and norms are unchanged; only the fp32 summation order of
// the user gradient differs (the REDs leave it unspecified as well).
// UBK + STAGED (SGD, when the staged rows fit shared memory; the launcher then provides the norm cache p.ub_norm): a claimed bucket's user
// rows are bulk-copied into shared memory with its first tile and read from there, and each touched row takes its SGD update when
// the bucket completes: every triple of user u is in u's bucket, so no other CTA reads p_u in the step.  The user norms that update
// needs are known before phase 1: the cache holds ||p_u||^2 and ||p_u||_1 of every user row (filled once per launch, rewritten
// by each update; an untouched row does not move under SGD), and the partition's histogram pass sums it over the batch.  gP and
// cntU are never written.  The cache also holds the item rows' norms, which the scatter pass sums over the batch's i and j, so
// phase 1 adds each occurrence's item regulariser to its gQ contribution; cntI is never written either, and phase 2 is the
// dense theta -= lr gQ over the item rows alone.
template <int VEC, int W, int NCH, bool GEN, class XCH, bool LEAN = false, bool UBK = false, bool STAGED = false>
__device__ __forceinline__ void bpr_steps_body(StepParams &p, XCH &xch)
{
    static_assert(!STAGED || UBK, "the staged form is a form of the user-bucketed mode");
    static_assert(!(GEN && LEAN), "the lean body is BPR only");
    static_assert(!UBK || (LEAN && VEC == 4 && !XCH::kActive), "the user-bucketed mode is a single-GPU lean mode");
    using RowOff = typename RowOffset<LEAN>::type;
    constexpr int GPW = 32 / W;                  // lane groups per warp
    constexpr int GROUPS = (kThreads / 32) * GPW;  // lane groups per CTA
    constexpr int UNR = (NCH * VEC <= (LEAN ? 8 : 4)) ? DRB_UNR : 1;  // triples in flight per group

    // index tiles: three planes u, i, j; UBK: kTileMax (u, i, j, 0) records
    __shared__ __align__(128) int32_t s_idx[2][UBK ? 4 : 3][kTileMax];
    __shared__ uint64_t s_bar[2];
    __shared__ union {
        double d[8][kThreads / 32];
        long long i[8][kThreads / 32];   // GEN && det: the fixed-point partials
    } s_red_u;
    double (&s_red)[8][kThreads / 32] = s_red_u.d;
    extern __shared__ __align__(16) unsigned char s_dyn[];   // UBK: partition histogram, then (staged rows +) bucket accumulator
    __shared__ int s_claim[3];                               // UBK: claimed bucket, its first and end position
    __shared__ unsigned s_wsum[kThreads / 32];               // UBK: per-warp sums of the bucket-count scan
    __shared__ int s_ucnt[kUbMaxRows], s_uoff[kUbMaxRows + 1];   // UBK: a tile's records per local user, their sorted offsets
    __shared__ uint16_t s_perm[kTileMax];                    // UBK: the tile's records in local-user order
    __shared__ float s_inv[3];                               // UBK, unorm: the step's inverse batch norms (u, i, j)

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int gl = lane % W, gw = lane / W;
    const int group = warp * GPW + gw;
    const int chunks = p.F / VEC;
    const int F = p.F;
    WsHeader *hdr = p.ws.hdr;

    if (tid == 0) {
        mbar_init(&s_bar[0], 1);
        mbar_init(&s_bar[1], 1);
        fence_mbar_init();
    }
    if constexpr (UBK)
        for (int k = tid; k < kUbMaxRows; k += kThreads) s_ucnt[k] = 0;   // each tile's sort leaves it zero again
    __syncthreads();
    if (*(volatile int *)&hdr->status != 0) return;   // split mode: a previous step already raised NaN
    uint32_t par0 = 0, par1 = 0;
    unsigned long long epoch = 0;
    const int tile = p.tile;
    const bool pw = GEN && p.loss >= DRB_LOSS_CL;   // point-wise: bj is the label plane, no negative row

    // stage one index tile: TMA bulk copy when full and 16-byte aligned, plain loads otherwise
    auto stage = [&](long long tbase, int cnt, int b) {
        const int32_t *su = p.bu + tbase, *si = p.bi + tbase, *sj = p.bj + tbase;
        bool bulk = (cnt % 4 == 0) && ((((uintptr_t)su | (uintptr_t)si | (uintptr_t)sj) & 15) == 0);
        if (bulk) {
            if (tid == 0) {
                uint32_t bytes = (uint32_t)cnt * 4u;
                mbar_expect_tx(&s_bar[b], 3u * bytes);
                tma_load_1d(&s_idx[b][0][0], su, bytes, &s_bar[b]);
                tma_load_1d(&s_idx[b][1][0], si, bytes, &s_bar[b]);
                tma_load_1d(&s_idx[b][2][0], sj, bytes, &s_bar[b]);
            }
        } else {
            for (int k = tid; k < cnt; k += kThreads) {
                s_idx[b][0][k] = __ldg(su + k);
                s_idx[b][1][k] = __ldg(si + k);
                s_idx[b][2][k] = __ldg(sj + k);
            }
            __syncthreads();
            if (tid == 0) mbar_arrive(&s_bar[b]);
        }
    };
    // UBK, thread 0: one bulk copy of the partitioned triples [t0, t0 + cnt) into tile buffer b (16-byte records: every start
    // and size is a multiple of 16 bytes)
    auto stage_ub = [&](int t0, int cnt, int b) {
        const uint32_t bytes = (uint32_t)cnt * 16u;
        mbar_expect_tx(&s_bar[b], bytes);
        tma_load_1d(&s_idx[b][0][0], p.ub_t + t0, bytes, &s_bar[b]);
    };
    // UBK, thread 0: claim the next non-empty bucket through the work counter, publish it in s_claim and stage its first tile;
    // dst != nullptr: its user rows join the same copy, into dst (row stride F)
    auto claim = [&](int b, float *dst) {
        int k, c0 = 0, c1 = 0;
        do {
            k = (int)atomicAdd(p.ub_count + 2 * p.ub_buckets, 1u);
            if (k < p.ub_buckets) { c0 = __ldcg(p.ub_range + 2 * k); c1 = __ldcg(p.ub_range + 2 * k + 1); }
        } while (k < p.ub_buckets && c0 == c1);
        s_claim[0] = k; s_claim[1] = c0; s_claim[2] = c1;
        if (k < p.ub_buckets) {
            asm volatile("fence.proxy.async.global;" ::: "memory");   // generic-proxy writes of the planes / rows -> bulk copy
            if (dst == nullptr) {
                stage_ub(c0, min(c1 - c0, kTileMax), b);
            } else {
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the slot's generic reads before its refill
                const int u0k = k * p.ub_users;
                const uint32_t rb = (uint32_t)min(p.ub_users, p.U - u0k) * (uint32_t)F * 4u, tb = (uint32_t)min(c1 - c0, kTileMax) * 16u;
                mbar_expect_tx(&s_bar[b], tb + rb);
                tma_load_1d(&s_idx[b][0][0], p.ub_t + c0, tb, &s_bar[b]);
                tma_load_1d(dst, p.P + (size_t)u0k * F, rb, &s_bar[b]);
            }
        }
    };
    // UBK + SGD with the norm cache: user rows staged and updated per bucket (see above); unorm: the cache is kept (regulariser on)
    constexpr bool ustage = UBK && STAGED;
    const bool unorm = ustage && ((p.reg1 != 0.f) || (p.reg2 != 0.f));
    auto mark = [&](long long s, int m) { if constexpr (ustage) phase_mark(s, m); };
    mark(0, 9);
    if constexpr (UBK) {
        if (unorm) {   // fill the norm cache: one pass over P and Q per launch (the item rows' entries follow the users')
            const long long nu = (long long)p.U * (W * NCH), nt = nu + (long long)p.I * (W * NCH);
            for (long long k0 = (long long)blockIdx.x * kThreads; k0 < nt; k0 += (long long)gridDim.x * kThreads) {
                const long long k = k0 + tid;
                const float4 *src = k < nu ? reinterpret_cast<const float4 *>(p.P) + k : reinterpret_cast<const float4 *>(p.Q) + (k - nu);
                const float4 v = k < nt ? __ldcg(src) : make_float4(0.f, 0.f, 0.f, 0.f);
                const float2 n = row_norms<W * NCH>(v);
                if (k < nt && k % (W * NCH) == 0) p.ub_norm[k / (W * NCH)] = n;
            }
            mark(0, 10);
            grid_barrier(&hdr->barrier, epoch);
            mark(0, 11);
        }
    }

    for (long long s = 0; s < p.n_steps; ++s) {
        const long long step = p.first_step + s;
        const long long base = p.step_offsets ? __ldg(p.step_offsets + step) : step * p.batch;
        const long long nb = p.step_offsets ? __ldg(p.step_offsets + step + 1) - base : min(p.batch, p.n - base);
        const long long ntiles = (nb + tile - 1) / tile;
        double *acc = hdr->acc[s & 1];
        const bool has_reg = (p.reg1 != 0.f) || (p.reg2 != 0.f);
        if constexpr (XCH::kActive) xch.begin_step(p, s, acc);   // item-side accumulators of this step's parity
        mark(s, 0);

        // ------------------------------------------------------------ phase 1
        if (p.phases & 1) {
        if (tid < 8 * (kThreads / 32)) {   // per-warp fp64 (GEN && det: int64) accumulators of this step
            if (GEN && p.det) (&s_red_u.i[0][0])[tid] = 0; else (&s_red[0][0])[tid] = 0.0;
        }
        bool det_ok = true;   // GEN && det: every value and addition of this step's fixed-point sums was in range
        __syncthreads();
        int buf = 0;
        long long t_i = blockIdx.x;
        // UBK: claimed bucket bk, its triples [r0, r1) in the partitioned records, position tt of the current tile; the gradient
        // rows and counts of its users u0 .. u0 + rows - 1 sum in s_gp / s_cu (row stride RS: F under ustage, 16-byte aligned
        // rows for the run sums; F + 1 otherwise, against bank conflicts between the groups of a warp in the per-triple atomics)
        int bk = 0, r0 = 0, r1 = 0, tt = 0, u0 = 0, rows = 0;
        const int RS = ustage ? F : F + 1;
        float *s_gp = nullptr;
        unsigned *s_cu = nullptr;
        float *s_rows = nullptr, *s_pu = nullptr;   // ustage: both row slots, the current bucket's slot
        int slot = 0;
        if constexpr (UBK) {
            const int NBK = p.ub_buckets, UBU = p.ub_users;
            unsigned *ucnt = p.ub_count, *ucur = p.ub_count + NBK;
            // ---- partition: per-CTA histogram of the bucket ids -> global counts
            unsigned *s_hist = reinterpret_cast<unsigned *>(s_dyn), *s_off = s_hist + NBK;
            for (int b = tid; b < NBK; b += kThreads) s_hist[b] = 0u;
            __syncthreads();
            const long long g0 = (long long)blockIdx.x * kThreads + tid, gstride = (long long)gridDim.x * kThreads;
            // the partition's passes take PB of a thread's triples at a time and issue all their global loads before using any:
            // one loop trip per triple waited out one round trip to L2 or HBM each (the norm-cache gathers are random).  The
            // thread's triples are still summed and placed in the order t, t + gstride, ...
            constexpr int PB = 4;
            float h_s2 = 0.f, h_l1 = 0.f;   // unorm: this thread's share of the batch's user norms, from the norm cache
            for (long long t0 = g0; t0 < nb; t0 += PB * gstride) {
                int u[PB];
                float2 n[PB];
#pragma unroll
                for (int q = 0; q < PB; ++q) {
                    const long long t = t0 + q * gstride;
                    u[q] = t < nb ? __ldg(p.bu + base + t) : -1;
                }
#pragma unroll
                for (int q = 0; q < PB; ++q) n[q] = (unorm && u[q] >= 0) ? __ldcg(p.ub_norm + u[q]) : make_float2(0.f, 0.f);
#pragma unroll
                for (int q = 0; q < PB; ++q) {
                    if (u[q] < 0) continue;
                    atomicAdd(&s_hist[u[q] / UBU], 1u);
                    if (unorm) {
                        h_s2 += n[q].x;
                        h_l1 += n[q].y;
                    }
                }
            }
            if (unorm) {
#pragma unroll
                for (int off = 16; off >= 1; off >>= 1) {
                    h_s2 += __shfl_xor_sync(0xffffffffu, h_s2, off);
                    h_l1 += __shfl_xor_sync(0xffffffffu, h_l1, off);
                }
                if (lane == 0) { s_red[4][warp] = (double)h_s2; s_red[1][warp] = (double)h_l1; }
            }
            __syncthreads();
            for (int b = tid; b < NBK; b += kThreads)
                if (s_hist[b] != 0u) red_add_u32(ucnt + b, s_hist[b]);
            if (unorm && (tid == 1 || tid == 4)) {   // l1u, s2u: one fp64 atomic per CTA; final after the next grid barrier
                double v = 0.0;
                for (int w = 0; w < kThreads / 32; ++w) { v += s_red[tid][w]; s_red[tid][w] = 0.0; }
                if (v != 0.0) atomicAdd(&acc[tid], v);
            }
            mark(s, 1);
            grid_barrier(&hdr->barrier, epoch);
            mark(s, 2);
            // each CTA reserves its slice of every bucket it holds triples of (s_hist becomes the slice's start within the bucket)
            // and copies the counts into s_off; eight buckets per thread at a time, their count loads and reservation atomics in
            // flight together.  Then an exclusive scan of the counts in every CTA; CTA 0 publishes the ranges.
            for (int bb = tid; bb < NBK; bb += 8 * kThreads) {
                unsigned c[8], r[8];
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const int b = bb + q * kThreads;
                    c[q] = 0u;
                    r[q] = 0u;
                    if (b < NBK) {
                        c[q] = __ldcg(ucnt + b);
                        const unsigned h = s_hist[b];
                        if (h != 0u) r[q] = atomicAdd(ucur + b, h);
                    }
                }
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const int b = bb + q * kThreads;
                    if (b < NBK) { s_off[b] = c[q]; s_hist[b] = r[q]; }
                }
            }
            __syncthreads();
            const int per = (NBK + kThreads - 1) / kThreads, b0 = min(NBK, tid * per), b1 = min(NBK, b0 + per);
            unsigned run = 0u;
            for (int b = b0; b < b1; ++b) run += s_off[b];
            unsigned incl = run;
#pragma unroll
            for (int off = 1; off < 32; off <<= 1) {
                const unsigned y = __shfl_up_sync(0xffffffffu, incl, off);
                if (lane >= off) incl += y;
            }
            if (lane == 31) s_wsum[warp] = incl;
            __syncthreads();
            unsigned start = incl - run;
            for (int w = 0; w < warp; ++w) start += s_wsum[w];
            for (int b = b0; b < b1; ++b) {
                const unsigned c = s_off[b];
                if (blockIdx.x == 0) { p.ub_range[2 * b] = (int)start; p.ub_range[2 * b + 1] = (int)(start + c); }
                s_off[b] = start + s_hist[b];
                s_hist[b] = 0u;
                start += c;
            }
            __syncthreads();
            mark(s, 3);
            // ---- scatter this CTA's triples into the partitioned records (the same triples as the histogram pass); a CTA holds
            // about two triples per bucket, so these stores land at random: one 16-byte store per triple, not three 4-byte ones
            // unorm: this pass also sums the item rows' cached norms over the batch (l1i, l1j, s2i, s2j)
            float h_in[4] = {0.f, 0.f, 0.f, 0.f};
            for (long long t0 = g0; t0 < nb; t0 += PB * gstride) {
                int u[PB], i[PB], j[PB];
                float2 ni[PB], nj[PB];
#pragma unroll
                for (int q = 0; q < PB; ++q) {
                    const long long t = t0 + q * gstride;
                    const bool ok = t < nb;
                    u[q] = ok ? __ldg(p.bu + base + t) : -1;
                    i[q] = ok ? __ldg(p.bi + base + t) : 0;
                    j[q] = ok ? __ldg(p.bj + base + t) : 0;
                }
#pragma unroll
                for (int q = 0; q < PB; ++q) {
                    const bool g = unorm && u[q] >= 0;
                    ni[q] = g ? __ldcg(p.ub_norm + p.U + i[q]) : make_float2(0.f, 0.f);
                    nj[q] = g ? __ldcg(p.ub_norm + p.U + j[q]) : make_float2(0.f, 0.f);
                }
#pragma unroll
                for (int q = 0; q < PB; ++q) {
                    if (u[q] < 0) continue;
                    const int b = u[q] / UBU;
                    const unsigned pos = s_off[b] + atomicAdd(&s_hist[b], 1u);
                    p.ub_t[pos] = make_int4(u[q], i[q], j[q], 0);
                    if (unorm) { h_in[0] += ni[q].y; h_in[1] += nj[q].y; h_in[2] += ni[q].x; h_in[3] += nj[q].x; }
                }
            }
            if (unorm) {
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    float v = h_in[q];
#pragma unroll
                    for (int off = 16; off >= 1; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
                    if (lane == 0) s_red[q < 2 ? 2 + q : 3 + q][warp] = (double)v;
                }
                __syncthreads();
                if (tid == 2 || tid == 3 || tid == 5 || tid == 6) {   // one fp64 atomic per CTA each; final after the barrier
                    double v = 0.0;
                    for (int w = 0; w < kThreads / 32; ++w) { v += s_red[tid][w]; s_red[tid][w] = 0.0; }
                    if (v != 0.0) atomicAdd(&acc[tid], v);
                }
            }
            asm volatile("fence.proxy.async.global;" ::: "memory");   // the records are read back by bulk copies (async proxy)
            mark(s, 4);
            grid_barrier(&hdr->barrier, epoch);
            for (long long k = g0; k < 2LL * NBK; k += gstride) ucnt[k] = 0u;   // counts, cursors: zero for the next step
            mark(s, 5);
            // ustage: two slots of UBU staged user rows (the current bucket's and the next one's) before the accumulator
            s_rows = reinterpret_cast<float *>(s_dyn);
            s_gp = s_rows + (ustage ? 2 * UBU * F : 0);
            s_cu = reinterpret_cast<unsigned *>(s_gp + UBU * RS);
            if (ustage && tid < 3) {   // as phase 2 derives them; read from shared memory where used (fewer live registers)
                const double n = unorm ? sqrt(((const volatile double *)acc)[tid + 4]) : 0.0;
                s_inv[tid] = n > 0 ? (float)(1.0 / n) : 0.f;
            }
            // ---- phase 1 over whole buckets, claimed dynamically (bucket sizes follow the user degrees)
            if (tid == 0) claim(0, ustage ? s_rows : nullptr);
            __syncthreads();
            bk = s_claim[0]; r0 = s_claim[1]; r1 = s_claim[2]; tt = r0;
        } else {
            if (t_i < ntiles) stage(base + t_i * tile, (int)min((long long)tile, nb - t_i * tile), 0);
        }
        for (; UBK ? bk < p.ub_buckets : t_i < ntiles; t_i += gridDim.x) {
            if constexpr (UBK) {
                if (tt == r0) {                                  // first tile of a bucket: zero its accumulator rows
                    u0 = bk * p.ub_users;
                    rows = min(p.ub_users, p.U - u0);
                    s_pu = s_rows + slot * p.ub_users * F;
                    for (int k = tid; k < rows * RS; k += kThreads) s_gp[k] = 0.f;
                    for (int k = tid; k < rows; k += kThreads) s_cu[k] = 0u;
                    __syncthreads();                             // zeroed; every thread has read s_claim
                }
                if (tid == 0) {                                  // prefetch: the bucket's next tile or the next bucket
                    if (tt + kTileMax < r1) stage_ub(tt + kTileMax, min(r1 - tt - kTileMax, kTileMax), buf ^ 1);
                    else claim(buf ^ 1, ustage ? s_rows + (slot ^ 1) * p.ub_users * F : nullptr);
                }
            } else {
                long long t_n = t_i + gridDim.x;
                if (t_n < ntiles) stage(base + t_n * tile, (int)min((long long)tile, nb - t_n * tile), buf ^ 1);
            }
            if (buf == 0) { mbar_wait(&s_bar[0], par0); par0 ^= 1; } else { mbar_wait(&s_bar[1], par1); par1 ^= 1; }
            const int cnt = UBK ? min(r1 - tt, kTileMax) : (int)min((long long)tile, nb - t_i * tile);
            // triple t's indices: xu[XS * t], xi[XS * t], xj[XS * t] (UBK: fields of record t)
            constexpr int XS = UBK ? 4 : 1;
            const int32_t *xu = s_idx[buf][0], *xi = UBK ? xu + 1 : s_idx[buf][1], *xj = UBK ? xu + 2 : s_idx[buf][2];
            float t_loss = 0.f, t_l1u = 0.f, t_l1i = 0.f, t_l1j = 0.f, t_s2u = 0.f, t_s2i = 0.f, t_s2j = 0.f, t_gb0 = 0.f;
            long long x_fx[7] = {0, 0, 0, 0, 0, 0, 0};   // GEN && det: the same seven sums, per triple in fixed point (det_acc)
            auto det_acc = [&](int k, float v) {
                x_fx[k] = det_add(x_fx[k], det_fix(v, k == 0 ? kDetAccScale : kDetNormScale, det_ok), det_ok);
            };
            // UBK + ustage: the tile's records are counting-sorted by local user into s_perm (user ul's run is
            // s_perm[s_uoff[ul] .. s_uoff[ul + 1])), and group g walks the sorted positions [lo, hi) = [g span, (g + 1) span), UNR
            // consecutive ones at a time.  It sums the user gradient of a run in registers (ua) and adds it to s_gp when the user
            // changes: with a plain read-add-write when the whole run lies in [lo, hi) (no other group holds it in this tile), with
            // shared-memory atomics when the run crosses a slice boundary (at most the first and the last run of a slice).  The
            // histogram is the tile's share of s_cu.  Without ustage (Adam, buckets too wide to stage: about one triple per user
            // and tile at the widths these run, where the sort costs more than it saves) the records are walked as in the plain
            // body, and each triple's user gradient and count are added with shared-memory atomics (row stride F + 1).
            int lo = 0, hi = 0, span = 0, urun = -1;
            constexpr bool sorted = UBK && STAGED;
            Vec<VEC> ua[NCH];
            if constexpr (UBK) {
                constexpr int PT = kTileMax / kThreads;   // records per thread
                if (sorted) {
                    int key[PT], rank[PT];
#pragma unroll
                    for (int q = 0; q < PT; ++q) {
                        const int k = tid + q * kThreads;
                        key[q] = k < cnt ? xu[XS * k] - u0 : 0;
                        rank[q] = k < cnt ? atomicAdd(&s_ucnt[key[q]], 1) : 0;
                    }
                    __syncthreads();
                    if (warp == 0) {   // exclusive scan of the counts; the counts join s_cu and are zeroed for the next tile
                        const int per = (rows + 31) / 32, b0 = min(rows, lane * per), b1 = min(rows, b0 + per);
                        int run = 0;
                        for (int b = b0; b < b1; ++b) run += s_ucnt[b];
                        int incl = run;
#pragma unroll
                        for (int off = 1; off < 32; off <<= 1) {
                            const int y = __shfl_up_sync(0xffffffffu, incl, off);
                            if (lane >= off) incl += y;
                        }
                        int start = incl - run;
                        for (int b = b0; b < b1; ++b) {
                            const int c = s_ucnt[b];
                            s_uoff[b] = start;
                            s_cu[b] += (unsigned)c;
                            s_ucnt[b] = 0;
                            start += c;
                        }
                        if (lane == 31) s_uoff[rows] = incl;
                    }
                    __syncthreads();
#pragma unroll
                    for (int q = 0; q < PT; ++q) {
                        const int k = tid + q * kThreads;
                        if (k < cnt) s_perm[s_uoff[key[q]] + rank[q]] = (uint16_t)k;
                    }
                    __syncthreads();
                    span = (cnt + GROUPS - 1) / GROUPS;   // every group takes the same trip count (pair_loss shuffles)
                    lo = min(cnt, group * span);
                    hi = min(cnt, lo + span);
                }
            }
            // UBK: add the run sum of local user urun to its accumulator row (every lane of the group, its own chunks)
            auto flush = [&]() {
                if (urun < 0) return;
                float *d = s_gp + urun * RS;
                const bool own = s_uoff[urun] >= lo && s_uoff[urun + 1] <= hi;
#pragma unroll
                for (int ch = 0; ch < NCH; ++ch) {
                    const int cc = gl + ch * W;
                    if (cc >= chunks) continue;
                    float4 *d4 = reinterpret_cast<float4 *>(d + cc * VEC);
                    if (own) {
                        float4 x = *d4;
                        x.x += ua[ch].v[0]; x.y += ua[ch].v[1]; x.z += ua[ch].v[2]; x.w += ua[ch].v[3];
                        *d4 = x;
                    } else {
#pragma unroll
                        for (int e = 0; e < VEC; ++e) atomicAdd(d + cc * VEC + e, ua[ch].v[e]);
                    }
                }
            };

            for (int tb = 0; tb < (sorted ? span : cnt); tb += (sorted ? UNR : GROUPS * UNR)) {
                Row<VEC, W, NCH> rp[UNR], rqi[UNR], rqj[UNR];
                int iu[UNR], ii[UNR], ij[UNR];
                RowOff ou[UNR], oi[UNR], oj[UNR];   // element offsets of the three rows (tables and accumulators alike)
                float lab[UNR];
                bool ok[UNR];
#pragma unroll
                for (int r = 0; r < UNR; ++r) {
                    int t = tb + r * GROUPS + group;
                    ok[r] = t < cnt;
                    if (sorted) {
                        ok[r] = lo + tb + r < hi;
                        t = ok[r] ? s_perm[lo + tb + r] : 0;
                    }
                    iu[r] = ok[r] ? xu[XS * t] : 0;
                    ii[r] = ok[r] ? xi[XS * t] : 0;
                    ij[r] = ok[r] ? xj[XS * t] : 0;
                    lab[r] = 0.f;
                    if (pw) {                       // label = batch[2].float() (MFRecommender.py:76); the j row stays zero
                        lab[r] = (float)ij[r];
                        ij[r] = 0;
                    }
                    if (!LEAN && p.neg_row_ptr != nullptr && ok[r]) {
                        const long long gt = base + t_i * tile + t;            // position of the triple in the planes
                        ij[r] = draw_negative(p, iu[r], (unsigned long long)gt, (unsigned long long)step);
                        if (p.neg_out != nullptr && gl == 0) p.neg_out[gt] = ij[r];
                    }
                    ou[r] = (RowOff)iu[r] * (RowOff)F;
                    oi[r] = (RowOff)ii[r] * (RowOff)F;
                    oj[r] = (RowOff)ij[r] * (RowOff)F;
                    bool staged = false;
                    if constexpr (UBK) {
                        if (ustage) {                        // the bucket's staged row (a quarter-warp reads one 128-byte segment)
                            staged = true;
                            const float *sr = s_pu + (ok[r] ? iu[r] - u0 : 0) * F;
#pragma unroll
                            for (int ch = 0; ch < NCH; ++ch) {
                                const int c = gl + ch * W;
                                float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
                                if (ok[r] && c < chunks) t = *reinterpret_cast<const float4 *>(sr + c * VEC);
                                rp[r].c[ch].v[0] = t.x; rp[r].c[ch].v[1] = t.y; rp[r].c[ch].v[2] = t.z; rp[r].c[ch].v[3] = t.w;
                            }
                        }
                    }
                    if (!staged) rp[r] = load_row<VEC, W, NCH>(p.P + ou[r], gl, chunks, ok[r]);
                    rqi[r] = load_row<VEC, W, NCH>(p.Q + oi[r], gl, chunks, ok[r]);
                    rqj[r] = load_row<VEC, W, NCH>(p.Q + oj[r], gl, chunks, ok[r] && !pw);
                }
                // scores of the UNR triples of this group (every lane of the group ends up with the same values)
                float ps[UNR], ns[UNR], cs[UNR], cn[UNR];
#pragma unroll
                for (int r = 0; r < UNR; ++r) {
                    ps[r] = dot_rows<VEC, W, NCH>(rp[r], rqi[r]);
                    ns[r] = dot_rows<VEC, W, NCH>(rp[r], rqj[r]);
                    if (GEN && p.bias != nullptr) {   // FM: pred += (u_bias(user) + i_bias(item)) + bias_  (FMRecommender.py:66-67)
                        const float ub = __ldcg(p.bias + iu[r]), b0 = __ldcg(p.bias + p.U + p.I);
                        ps[r] += (ub + __ldcg(p.bias + p.U + ii[r])) + b0;
                        ns[r] += (ub + __ldcg(p.bias + p.U + ij[r])) + b0;
                    }
                    if (pw) ns[r] = lab[r];         // pair_loss receives the label in place of the negative score
                }
                // The scalar chain (sigmoid -> log -> coefficient, ~40 instructions) would be replayed by all W lanes for
                // each of the UNR triples; instead lane gl evaluates it ONCE, for triple (gl % UNR) of its group, and the
                // coefficients d(loss)/d(pos), d(loss)/d(neg) are handed round with shuffles.
                auto pair_loss = [&](float pos, float neg, float &c_pos, float &c_neg) -> float {
                    if (GEN && p.loss == DRB_LOSS_CL) {     // BCEWithLogitsLoss(sum): (1-y) x - log_sigmoid(x), neg = y
                        const float z = expf(-fabsf(pos));
                        const float logsig = fminf(pos, 0.f) - log1pf(z);
                        const float dls = pos < 0.f ? 1.f - z / (1.f + z) : z / (1.f + z);
                        c_pos = (1.f - neg) - dls;
                        c_neg = 0.f;
                        return (1.f - neg) * pos - logsig;
                    }
                    if (GEN && p.loss == DRB_LOSS_SL) {     // MSELoss(sum): (x - y)^2, neg = y
                        const float d = pos - neg;
                        c_pos = 2.f * d;
                        c_neg = 0.f;
                        return d * d;
                    }
                    if (GEN && p.loss == DRB_LOSS_HL) {     // clamp(1 - (pos - neg), min=0); clamp's backward passes at equality
                        const float m = 1.f - (pos - neg);
                        c_pos = (m >= 0.f) ? -1.f : 0.f;
                        c_neg = -c_pos;
                        return m > 0.f ? m : 0.f;
                    }
                    if (GEN && p.loss == DRB_LOSS_TL) {     // sigmoid(neg - pos) + sigmoid(neg^2)
                        const float s1 = 1.f / (1.f + expf(-(neg - pos))), s2 = 1.f / (1.f + expf(-(neg * neg)));
                        c_pos = -(s1 * (1.f - s1));
                        c_neg = s1 * (1.f - s1) + s2 * (1.f - s2) * 2.f * neg;
                        return s1 + s2;
                    }
                    const float x = pos - neg;
                    // deterministic mode: exp in fp64, rounded once -- the correctly rounded expf of the host's libm, so the
                    // coefficient (it scales every contribution of the triple) is the fp64 oracle's to the bit
                    const float ex = (GEN && p.det) ? (float)exp(-(double)x) : expf(-x);
                    const float sg = 1.f / (1.f + ex);
                    c_pos = -(sg * (1.f - sg)) / (1e-10f + sg);
                    c_neg = -c_pos;
                    return -logf(1e-10f + sg);
                };
                if constexpr (W >= UNR) {
                    float p_own = ps[0], n_own = ns[0];
                    bool ok_own = ok[0];
#pragma unroll
                    for (int r = 1; r < UNR; ++r)
                        if ((gl % UNR) == r) { p_own = ps[r]; n_own = ns[r]; ok_own = ok[r]; }
                    float cp_own, cn_own;
                    const float l_own = pair_loss(p_own, n_own, cp_own, cn_own);
                    if (gl < UNR && ok_own) {
                        if (GEN && p.det) det_acc(0, l_own); else t_loss += l_own;
                    }
#pragma unroll
                    for (int r = 0; r < UNR; ++r) {
                        cs[r] = __shfl_sync(0xffffffffu, cp_own, (lane - gl) + r);
                        cn[r] = GEN ? __shfl_sync(0xffffffffu, cn_own, (lane - gl) + r) : -cs[r];
                    }
                } else {
#pragma unroll
                    for (int r = 0; r < UNR; ++r) {
                        const float l = pair_loss(ps[r], ns[r], cs[r], cn[r]);
                        if (gl == 0 && ok[r]) {
                            if (GEN && p.det) det_acc(0, l); else t_loss += l;
                        }
                    }
                }
#pragma unroll
                for (int r = 0; r < UNR; ++r) {
                    if (!ok[r]) continue;
                    const float c = cs[r];
                    if (has_reg && !unorm) {   // unorm: the partition has summed the batch norms from the norm cache
                        float l1u = 0, l1i = 0, l1j = 0, s2u = 0, s2i = 0, s2j = 0;
                        Row<VEC, W, NCH> nu_ = rp[r], ni_ = rqi[r], nj_ = rqj[r];
                        if (!LEAN && p.Pn != nullptr) {   // regulariser on the ego rows (LightGCNRecommender.py:145-146,159)
                            nu_ = load_row<VEC, W, NCH>(p.Pn + ou[r], gl, chunks, true);
                            ni_ = load_row<VEC, W, NCH>(p.Qn + oi[r], gl, chunks, true);
                            nj_ = load_row<VEC, W, NCH>(p.Qn + oj[r], gl, chunks, true);
                        }
#pragma unroll
                        for (int ch = 0; ch < NCH; ++ch)
#pragma unroll
                            for (int e = 0; e < VEC; ++e) {
                                float a = nu_.c[ch].v[e], b = ni_.c[ch].v[e], d = nj_.c[ch].v[e];
                                l1u += fabsf(a); s2u = fmaf(a, a, s2u);
                                l1i += fabsf(b); s2i = fmaf(b, b, s2i);
                                l1j += fabsf(d); s2j = fmaf(d, d, s2j);
                            }
                        if (GEN && p.det) {
                            det_acc(1, l1u); det_acc(2, l1i); det_acc(3, l1j);
                            det_acc(4, s2u); det_acc(5, s2i); det_acc(6, s2j);
                        } else {
                            t_l1u += l1u; t_s2u += s2u;
                            t_l1i += l1i; t_l1j += l1j;
                            t_s2i += s2i; t_s2j += s2j;
                        }
                    }
                    if (p.apply) {
                        if constexpr (UBK && STAGED) {
                            if (iu[r] - u0 != urun) {   // a new run: flush the last one
                                flush();
                                urun = iu[r] - u0;
#pragma unroll
                                for (int ch = 0; ch < NCH; ++ch)
#pragma unroll
                                    for (int e = 0; e < VEC; ++e) ua[ch].v[e] = 0.f;
                            }
                        }
#pragma unroll
                        for (int ch = 0; ch < NCH; ++ch) {
                            int cc = gl + ch * W;
                            if (cc >= chunks) continue;
                            Vec<VEC> gu, gi, gj;
#pragma unroll
                            for (int e = 0; e < VEC; ++e) {
                                if (!GEN || p.loss == DRB_LOSS_BPR) {   // c_neg == -c_pos: the reference's BPR arithmetic
                                    gu.v[e] = c * (rqi[r].c[ch].v[e] - rqj[r].c[ch].v[e]);
                                    gi.v[e] = c * rp[r].c[ch].v[e];
                                    gj.v[e] = -gi.v[e];
                                    if (UBK && unorm) {   // the item rows' regulariser, once per occurrence (no counters)
                                        gi.v[e] += reg_term(rqi[r].c[ch].v[e], s_inv[1], p);
                                        gj.v[e] += reg_term(rqj[r].c[ch].v[e], s_inv[2], p);
                                    }
                                } else {
                                    gu.v[e] = c * rqi[r].c[ch].v[e] + cn[r] * rqj[r].c[ch].v[e];
                                    gi.v[e] = c * rp[r].c[ch].v[e];
                                    gj.v[e] = cn[r] * rp[r].c[ch].v[e];
                                }
                            }
                            if (GEN && p.det) {
#pragma unroll
                                for (int e = 0; e < VEC; ++e) {
                                    det_red(p.ws.gP64 + ou[r] + cc * VEC + e, gu.v[e], det_ok);
                                    det_red(p.ws.gQ64 + oi[r] + cc * VEC + e, gi.v[e], det_ok);
                                    if (!pw) det_red(p.ws.gQ64 + oj[r] + cc * VEC + e, gj.v[e], det_ok);
                                }
                            } else {
                                if constexpr (UBK && STAGED) {
#pragma unroll
                                    for (int e = 0; e < VEC; ++e) ua[ch].v[e] += gu.v[e];
                                } else if constexpr (UBK) {
                                    float *d = s_gp + (iu[r] - u0) * RS + cc * VEC;
#pragma unroll
                                    for (int e = 0; e < VEC; ++e) atomicAdd(d + e, gu.v[e]);
                                } else {
                                    red_row<VEC>(p.ws.gP + ou[r] + cc * VEC, gu);
                                }
                                red_row<VEC>(p.ws.gQ + oi[r] + cc * VEC, gi);
                                if (!pw) red_row<VEC>(p.ws.gQ + oj[r] + cc * VEC, gj);
                            }
                        }
                        if (gl == 0) {
                            if constexpr (UBK) {
                                if (!sorted) atomicAdd(s_cu + (iu[r] - u0), 1u);   // sorted: the tile's sort has counted it
                            } else if (GEN && p.U == 0) {
                                red_add_u64(p.ws.cntI + iu[r], 1ull);
                            } else {
                                red_add_u32(p.ws.cntU + iu[r], 1u);
                            }
                            if (!(UBK && ustage)) {   // ustage: the item sweep needs no counters
                                red_add_u64(p.ws.cntI + ii[r], 1ull);
                                if (!pw) red_add_u64(p.ws.cntI + ij[r], 1ull << 32);
                            }
                            if (GEN && p.bias != nullptr) {   // d loss / d (u_bias, i_bias, bias_): no regulariser (:76-95)
                                const float cboth = pw ? c : c + cn[r];
                                asm volatile("red.relaxed.gpu.global.add.f32 [%0], %1;" ::"l"(p.ws.gB + iu[r]), "f"(cboth) : "memory");
                                asm volatile("red.relaxed.gpu.global.add.f32 [%0], %1;" ::"l"(p.ws.gB + p.U + ii[r]), "f"(c) : "memory");
                                if (!pw)
                                    asm volatile("red.relaxed.gpu.global.add.f32 [%0], %1;" ::"l"(p.ws.gB + p.U + ij[r]), "f"(cn[r]) : "memory");
                                t_gb0 += cboth;
                            }
                        }
                    }
                }
            }
            if constexpr (UBK && STAGED) flush();
            // per-thread fp32 partials cover <= tile/GROUPS triples: warp-reduce, widen to fp64 in smem
            // (GEN && det: the fixed-point partials are summed as integers, in the same smem slots; FM's biases never run det)
            {
                float tv[8] = {t_loss, t_l1u, t_l1i, t_l1j, t_s2u, t_s2i, t_s2j, t_gb0};
                const int nv = has_reg ? 7 : 1;
                for (int k = 0; k < 8; ++k) {
                    if (k >= nv && !(GEN && k == 7 && p.bias != nullptr)) continue;
                    if (GEN && p.det && k < 7) {
                        long long v = x_fx[k];
#pragma unroll
                        for (int off = 16; off >= 1; off >>= 1) v = det_add(v, __shfl_xor_sync(0xffffffffu, v, off), det_ok);
                        if (lane == 0) s_red_u.i[k][warp] = det_add(s_red_u.i[k][warp], v, det_ok);
                        continue;
                    }
                    float v = tv[k];
#pragma unroll
                    for (int off = 16; off >= 1; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
                    if (lane == 0) s_red[k][warp] += (double)v;
                }
            }
            __syncthreads();  // tile buffer free for re-staging
            buf ^= 1;
            if constexpr (UBK) {
                tt += kTileMax;
                if (tt >= r1 && ustage) {
                    // the bucket is complete: each touched row takes its SGD update from the staged row and is stored back, with
                    // its new norms (one chunk per thread, the W * NCH chunks of a row on consecutive lanes); untouched rows stay
                    constexpr int CH = W * NCH;
                    const int n = rows * CH;
                    for (int k0 = 0; k0 < n; k0 += kThreads) {
                        const int k = k0 + tid, r = k / CH, c = k - r * CH;
                        const bool live = k < n && s_cu[r] != 0u;
                        float4 th = make_float4(0.f, 0.f, 0.f, 0.f);
                        if (live) {
                            const float *a = s_pu + r * F + c * VEC, *g = s_gp + r * F + c * VEC;
                            const float cnt = (float)s_cu[r];
                            th.x = a[0] - p.lr * reg_grad(a[0], p.gscale * g[0], cnt, s_inv[0], 0.f, 0.f, p);
                            th.y = a[1] - p.lr * reg_grad(a[1], p.gscale * g[1], cnt, s_inv[0], 0.f, 0.f, p);
                            th.z = a[2] - p.lr * reg_grad(a[2], p.gscale * g[2], cnt, s_inv[0], 0.f, 0.f, p);
                            th.w = a[3] - p.lr * reg_grad(a[3], p.gscale * g[3], cnt, s_inv[0], 0.f, 0.f, p);
                            __stcg(reinterpret_cast<float4 *>(p.P + (size_t)(u0 + r) * F + c * VEC), th);
                        }
                        if (unorm) {
                            const float2 nrm = row_norms<CH>(th);
                            if (live && c == 0) __stcg(p.ub_norm + u0 + r, nrm);
                        }
                    }
                    __syncthreads();   // slot and accumulator free; s_claim holds the bucket claimed during this tile
                    bk = s_claim[0]; r0 = s_claim[1]; r1 = s_claim[2]; tt = r0;
                    slot ^= 1;
                } else if (tt >= r1) {   // the bucket is complete: one plain store per touched row and counter; untouched rows keep zeros
                    for (int k = tid; k < rows * chunks; k += kThreads) {
                        const int r = k / chunks, c = k - r * chunks;
                        if (s_cu[r] == 0u) continue;
                        const float *a = s_gp + r * RS + c * VEC;
                        __stcg(reinterpret_cast<float4 *>(p.ws.gP + (size_t)(u0 + r) * F + c * VEC), make_float4(a[0], a[1], a[2], a[3]));
                    }
                    for (int k = tid; k < rows; k += kThreads)
                        if (s_cu[k] != 0u) __stcg(p.ws.cntU + u0 + k, s_cu[k]);
                    __syncthreads();   // accumulator free; s_claim holds the bucket claimed during this tile
                    bk = s_claim[0]; r0 = s_claim[1]; r1 = s_claim[2]; tt = r0;
                }
            }
        }
        // CTA reduction of the 7 partial sums -> one fp64 atomic each
        __syncthreads();
        if (tid < (has_reg ? 7 : 1) || (GEN && tid == 7 && p.bias != nullptr)) {
            if (GEN && p.det) {
                long long v = 0;
                for (int w = 0; w < kThreads / 32; ++w) v = det_add(v, s_red_u.i[tid][w], det_ok);
                if (v != 0) {
                    const long long old = (long long)atomicAdd(reinterpret_cast<unsigned long long *>(p.ws.accfx + tid),
                                                               (unsigned long long)v);
                    det_add(old, v, det_ok);
                }
            } else {
                double v = 0;
                for (int w = 0; w < kThreads / 32; ++w) v += s_red[tid][w];
                if (v != 0.0) atomicAdd(&acc[tid], v);
            }
        }
        // GEN && det: a value or sum out of range anywhere in the CTA flags the step in accfx[7] (a slot FM's bias sum would use;
        // FM never runs det), read back before phase 2
        if (GEN && p.det)
            if (!__syncthreads_and(det_ok) && tid == 0) red_add_u64(reinterpret_cast<unsigned long long *>(p.ws.accfx + 7), 1ull);
        }  // phase 1
        mark(s, 6);
        if (p.phases == 3) grid_barrier(&hdr->barrier, epoch);
        mark(s, 7);
        if constexpr (UBK)
            if (blockIdx.x == 0 && tid == 0) p.ub_count[2 * p.ub_buckets] = 0u;   // every claim of this step is done
        if (!(p.phases & 2)) break;   // split mode: the host reduces gQ / counters / acc across ranks now
        if (GEN && p.det) {
            // fixed-point scalar sums -> acc (the table sums stay in fixed point: the DET sweep reads and clears them); a flagged
            // step gets a NaN loss, which every CTA sees after the barrier and which stops the launch before phase 2
            if (blockIdx.x == 0 && tid == 0) {
                const bool flagged = __ldcg(p.ws.accfx + 7) != 0;
                for (int k = 0; k < 8; ++k) {
                    acc[k] = (k == 0 && flagged) ? __longlong_as_double(0x7ff8000000000000ll)
                                                 : (double)__ldcg(p.ws.accfx + k) / (k == 0 ? kDetAccScale : kDetNormScale);
                    __stcg(p.ws.accfx + k, 0ll);
                }
            }
            grid_barrier(&hdr->barrier, epoch);
        }
        if constexpr (XCH::kActive) {
            // rendezvous with the other ranks; acc[0..7] become the GLOBAL sums (identical on every rank)
            if (!xch.after_phase1(p, s, acc, epoch)) break;
        }

        // ------------------------------------------------------------ phase 2
        double bpr, l1u, l1i, l1j, s2u, s2i, s2j;
        {
            const volatile double *va = acc;
            bpr = va[0]; l1u = va[1]; l1i = va[2]; l1j = va[3]; s2u = va[4]; s2i = va[5]; s2j = va[6];
        }
        double nu = sqrt(s2u), ni = sqrt(s2i), nj = sqrt(s2j);
        // fp32 assembly of the scalar loss, in the reference's order (MFRecommender.py:88-95)
        float loss = (float)bpr;
        loss += p.reg1 * ((float)l1i + (float)l1j);
        loss += p.reg2 * ((float)ni + (float)nj);
        loss += p.reg1 * (float)l1u;
        loss += p.reg2 * (float)nu;
        if (blockIdx.x == 0 && tid == 0) p.step_loss[s] = (double)loss;
        if constexpr (!XCH::kActive)
            if (blockIdx.x == 0 && tid < 8) hdr->acc[(s + 1) & 1][tid] = 0.0;  // recycle the other accumulator
        if (isnan(loss)) {
            if (blockIdx.x == 0 && tid == 0) {
                hdr->status = DRB_ERR_NAN_LOSS;
                hdr->nan_step = step;
            }
            break;  // uniform across the grid: every CTA computed the same loss
        }
        if (p.apply) {
            Norms nm;
            nm.inv_u = nu > 0 ? (float)(1.0 / nu) : 0.f;
            nm.inv_i = ni > 0 ? (float)(1.0 / ni) : 0.f;
            nm.inv_j = nj > 0 ? (float)(1.0 / nj) : 0.f;
            AdamCoef ac;
            ac.step_size = 0.f;
            ac.bc2_sqrt = 1.f;
            if (p.opt == DRB_OPT_ADAM) {
                double t = (double)(p.adam_step0 + s + 1);
                ac.step_size = (float)((double)p.lr / (1.0 - pow((double)p.beta1, t)));
                ac.bc2_sqrt = (float)sqrt(1.0 - pow((double)p.beta2, t));
            }
            const bool dense = (GEN && p.det) || (p.dense_hint >= 0 ? (p.dense_hint != 0)
                                                                 : ((p.opt != DRB_OPT_SGD) || (3 * nb >= ((long long)p.U + p.I) / 4)));
            if constexpr (XCH::kActive) {
                // this rank's item slice: reduce the ranks' accumulators, update, broadcast the new rows; then the local user
                // rows are swept below with the item half switched off (p.I = 0 inside the policy's copy of the parameters)
                xch.template item_slice<VEC, W, NCH>(p, s, nm, ac, gl, group, GROUPS, chunks, epoch);
            }
            if (GEN && p.det) {                    // single GPU only (launch_steps): no exchange policy is active here
                if constexpr (GEN && !XCH::kActive) {
                    if (p.opt == DRB_OPT_SGD)
                        dense_sweep<VEC, W, NCH, DRB_OPT_SGD, false, true>(p, nm, ac, gl, group, GROUPS, chunks);
                    else if (p.opt == DRB_OPT_ADAM)
                        dense_sweep<VEC, W, NCH, DRB_OPT_ADAM, false, true>(p, nm, ac, gl, group, GROUPS, chunks);
                    else if (p.opt == DRB_OPT_ADAGRAD)
                        dense_sweep<VEC, W, NCH, DRB_OPT_ADAGRAD, false, true>(p, nm, ac, gl, group, GROUPS, chunks);
                    else
                        dense_sweep<VEC, W, NCH, DRB_OPT_RMSPROP, false, true>(p, nm, ac, gl, group, GROUPS, chunks);
                }
            } else if (UBK && ustage) {
                // the user rows took their update when their bucket completed, and phase 1 has added the item regulariser to
                // gQ: every item row takes theta -= lr gQ (a zero chunk does not move), one chunk per thread, and rewrites its
                // norm cache entry (the W * NCH chunks of a row on consecutive lanes)
                constexpr int CH = W * NCH;
                const long long nt = (long long)p.I * CH;
                for (long long k0 = (long long)blockIdx.x * kThreads; k0 < nt; k0 += (long long)gridDim.x * kThreads) {
                    const long long k = k0 + tid;
                    float4 th = make_float4(0.f, 0.f, 0.f, 0.f), g = th;
                    float4 *tp = reinterpret_cast<float4 *>(p.Q) + k, *gp = reinterpret_cast<float4 *>(p.ws.gQ) + k;
                    if (k < nt) { th = __ldcg(tp); g = __ldcg(gp); }
                    if (g.x != 0.f || g.y != 0.f || g.z != 0.f || g.w != 0.f) {
                        th.x = th.x - p.lr * g.x; th.y = th.y - p.lr * g.y; th.z = th.z - p.lr * g.z; th.w = th.w - p.lr * g.w;
                        __stcg(tp, th);
                        __stcg(gp, make_float4(0.f, 0.f, 0.f, 0.f));
                    }
                    if (unorm) {
                        const float2 nrm = row_norms<CH>(th);
                        if (k < nt && k % CH == 0) __stcg(p.ub_norm + p.U + k / CH, nrm);
                    }
                }
            } else if (dense || p.opt != DRB_OPT_SGD) {   // stateful optimisers always sweep (claim mode is SGD only)
                if (p.opt == DRB_OPT_SGD)
                    dense_sweep<VEC, W, NCH, DRB_OPT_SGD, XCH::kActive>(p, nm, ac, gl, group, GROUPS, chunks);
                else if (p.opt == DRB_OPT_ADAM)
                    dense_sweep<VEC, W, NCH, DRB_OPT_ADAM, XCH::kActive>(p, nm, ac, gl, group, GROUPS, chunks);
                else if constexpr (GEN) {          // launch_steps routes these two to the GEN instantiation
                    if (p.opt == DRB_OPT_ADAGRAD)
                        dense_sweep<VEC, W, NCH, DRB_OPT_ADAGRAD>(p, nm, ac, gl, group, GROUPS, chunks);
                    else
                        dense_sweep<VEC, W, NCH, DRB_OPT_RMSPROP>(p, nm, ac, gl, group, GROUPS, chunks);
                }
            } else {
                // claim mode (SGD only): the first group to swap a row's counter to zero applies it
                for (long long t0 = (long long)blockIdx.x * tile; t0 < nb; t0 += (long long)gridDim.x * tile) {
                    const int cnt = (int)min((long long)tile, nb - t0);
                    for (int tb = 0; tb < cnt; tb += GROUPS) {
                        int t = tb + group;
                        bool ok = t < cnt;
                        int u = 0, i = 0, j = 0;
                        if (ok) {
                            u = __ldg(p.bu + base + t0 + t);
                            i = __ldg(p.bi + base + t0 + t);
                            j = pw ? i : __ldg(p.bj + base + t0 + t);   // point-wise: that plane holds labels
                        }
                        unsigned cu = 0;
                        unsigned long long ci = 0, cj = 0;
                        if (ok && gl == 0) {
                            cu = atomicExch(p.ws.cntU + u, 0u);
                            ci = atomicExch(p.ws.cntI + i, 0ull);
                            cj = atomicExch(p.ws.cntI + j, 0ull);
                        }
                        cu = __shfl_sync(0xffffffffu, cu, gw * W);
                        ci = __shfl_sync(0xffffffffu, ci, gw * W);
                        cj = __shfl_sync(0xffffffffu, cj, gw * W);
                        if (cu != 0) {
                            size_t o = (size_t)u * F;
                            apply_row<VEC, W, NCH, DRB_OPT_SGD>(p.P + o, p.ws.gP + o, nullptr, nullptr, gl, chunks, (float)cu,
                                                                nm.inv_u, 0.f, 0.f, p, ac, true);
                        }
                        if (ci != 0) {
                            size_t o = (size_t)i * F;
                            apply_row<VEC, W, NCH, DRB_OPT_SGD>(p.Q + o, p.ws.gQ + o, nullptr, nullptr, gl, chunks,
                                                                (float)(unsigned)(ci & 0xffffffffull), nm.inv_i,
                                                                (float)(unsigned)(ci >> 32), nm.inv_j, p, ac, true);
                        }
                        if (cj != 0) {
                            size_t o = (size_t)j * F;
                            apply_row<VEC, W, NCH, DRB_OPT_SGD>(p.Q + o, p.ws.gQ + o, nullptr, nullptr, gl, chunks,
                                                                (float)(unsigned)(cj & 0xffffffffull), nm.inv_i,
                                                                (float)(unsigned)(cj >> 32), nm.inv_j, p, ac, true);
                        }
                    }
                }
            }
        }
        if (GEN && p.apply && p.bias != nullptr) {
            // FM's U + I + 1 first-order scalars: the same optimiser switch, no regulariser; the accumulator is cleared
            const double gb0 = ((const volatile double *)acc)[7];
            float step_size = 0.f, bc2_sqrt = 1.f;
            if (p.opt == DRB_OPT_ADAM) {
                double t = (double)(p.adam_step0 + s + 1);
                step_size = (float)((double)p.lr / (1.0 - pow((double)p.beta1, t)));
                bc2_sqrt = (float)sqrt(1.0 - pow((double)p.beta2, t));
            }
            const long long nbias = (long long)p.U + p.I + 1;
            for (long long k = (long long)blockIdx.x * kThreads + tid; k < nbias; k += (long long)gridDim.x * kThreads) {
                const float g = (k == nbias - 1) ? (float)gb0 : __ldcg(p.ws.gB + k);
                float th = __ldcg(p.bias + k);
                if (p.opt == DRB_OPT_SGD) {
                    th = th - p.lr * g;
                } else if (p.opt == DRB_OPT_ADAGRAD) {
                    const float ss = __ldcg(p.ws.mB + k) + g * g;
                    th = th - p.lr * (g / (sqrtf(ss) + 1e-10f));
                    __stcg(p.ws.mB + k, ss);
                } else if (p.opt == DRB_OPT_RMSPROP) {
                    const float sq = __ldcg(p.ws.mB + k) * 0.99f + (1.f - 0.99f) * g * g;
                    th = th - p.lr * (g / (sqrtf(sq) + 1e-8f));
                    __stcg(p.ws.mB + k, sq);
                } else {
                    float mm = __ldcg(p.ws.mB + k), vv = __ldcg(p.ws.vB + k);
                    mm = mm + (g - mm) * (1.f - p.beta1);
                    vv = vv * p.beta2 + (1.f - p.beta2) * g * g;
                    th = th - step_size * (mm / (sqrtf(vv) / bc2_sqrt + p.eps));
                    __stcg(p.ws.mB + k, mm);
                    __stcg(p.ws.vB + k, vv);
                }
                __stcg(p.bias + k, th);
                if (k != nbias - 1 && g != 0.f) __stcg(p.ws.gB + k, 0.f);
            }
        }
        mark(s, 8);
        if constexpr (XCH::kActive) {
            if (!xch.end_step(p, s, epoch)) break;   // every rank's item slice has landed in this rank's replica
        } else {
            if (s + 1 < p.n_steps) grid_barrier(&hdr->barrier, epoch);
        }
    }
}

template <int VEC, int W, int NCH, bool GEN>
__global__ void __launch_bounds__(kThreads, DRB_MINB) mf_bpr_steps_kernel(StepParams p)
{
    NoExchange x;
    bpr_steps_body<VEC, W, NCH, GEN, NoExchange>(p, x);
}

template <int VEC, int W, int NCH, bool UBK = false, bool STAGED = false>
__global__ void __launch_bounds__(kThreads, DRB_MINB) mf_bpr_steps_lean_kernel(StepParams p)
{
    NoExchange x;
    bpr_steps_body<VEC, W, NCH, false, NoExchange, true, UBK, STAGED>(p, x);
}

// the conditions under which the lean body computes what the general one does
inline bool step_params_lean(const StepParams &p)
{
    return p.loss == DRB_LOSS_BPR && p.opt <= DRB_OPT_ADAM && p.bias == nullptr && p.det == 0 && p.Pn == nullptr &&
           p.Qn == nullptr && p.neg_row_ptr == nullptr && (unsigned long long)p.U * (unsigned)p.F < (1ull << 32) &&
           (unsigned long long)p.I * (unsigned)p.F < (1ull << 32);
}


}  // namespace drb
