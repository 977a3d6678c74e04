// randperm.cu -- the DataLoader's epoch permutation, bit for bit, on the device.
//
// Stands behind `DataLoader(BasicDataset(samples), batch_size, shuffle=True)` of run_examples/test.py:93-94 /
// daisy/utils/dataset.py:5-8: RandomSampler.__iter__ seeds a private CPU generator and yields
// torch.randperm(n, generator) -- ATen's randperm_cpu, which for n < 2^32 / 20 is the textbook Fisher-Yates walk
//     A = arange(n);  for i in 0 .. n-2:  z = mt19937() % (n - i);  swap(A[i], A[i + z])
// driven by the 32-bit outputs of MT19937 seeded with init_genrand(seed & 0xffffffff).  At 80 M triples that walk costs
// the reference-exact path of fit() 2.3 s per epoch on the host (against 19 ms of training), so it is rebuilt here:
//
//   mt19937_stream_kernel   ONE CTA regenerates the 624-word state in the three data-parallel phases the recurrence
//                           x[k+624] = x[k+397] ^ twist(x[k], x[k+1]) allows (0..226 | 227..453 | 454..623) and streams the
//                           tempered words to HBM: the sequence is inherently sequential across 624-word blocks, parallel
//                           inside one (about 0.2 us per block).
//   mt19937_segments_kernel the same stream from MANY CTAs: CTA k jumps the seeded state ahead by k segments of 1 680 blocks with
//                           precomputed jump polynomials (GF(2)-linear jump-ahead, see below) and regenerates only its segment.
//                           Used after a one-off device check against the one-CTA kernel; that one stays as the fallback.
//   fisher_yates_kernel     the SAME permutation as the sequential walk, computed in parallel with deterministic
//                           reservations (Shun, Gu, Blelloch, Fineman, Gibbons: "Sequential random permutation, list
//                           contraction and tree contraction are highly parallel", SODA 2015): iteration i touches cells i
//                           and h(i) = i + w_i % (n - i).  Each round takes the earliest unfinished iterations (the failed
//                           ones of the round before + a fresh window of 1/8 of what is left), every iteration writes its
//                           index into both of its cells with atomicMin, and the iterations that own both cells swap; an
//                           iteration commits only when no earlier unfinished iteration shares a cell with it, so the
//                           result equals the sequential order.  ~70 rounds for 80 M elements, 1.2 n cell visits, one
//                           persistent cooperative launch (two grid barriers per round).
// Integer kernels: bit-exact by construction; tests compare against torch.randperm itself.
#include <stdlib.h>
#include <string.h>

#include <mutex>
#include <vector>

#include "common.cuh"

namespace drb {

constexpr int kMtN = 624, kMtM = 397;

__device__ __forceinline__ uint32_t mt_twist(uint32_t a, uint32_t b)
{
    const uint32_t y = (a & 0x80000000u) | (b & 0x7fffffffu);
    return (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
}
__device__ __forceinline__ uint32_t mt_temper(uint32_t y)
{
    y ^= (y >> 11);
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= (y >> 18);
    return y;
}

// out[0..n) = the first n outputs of at::mt19937(seed) (== numpy's init_genrand + genrand_int32).
// One CTA; thread t (t < 227) owns the state words t, t+227 and t+454 (t < 170).  In the sequential walk
//   x[k]     = x[k+397] ^ twist(x[k], x[k+1])                 k in [0, 227)    -- all inputs are OLD words
//   x[k]     = x[k-227] ^ twist(x[k], x[k+1])                 k in [227, 454)  -- x[k-227] is thread t's own NEW word
//   x[k]     = x[k-227] ^ twist(x[k], x[k+1])                 k in [454, 623)  -- likewise
//   x[623]   = x[396]   ^ twist(x[623], x[0])                                   -- NEW x[0]: recomputed by its reader
// every OLD input can be read before anything is written, and every NEW input is a register of the same thread.  So a
// 624-word block costs: load the old words, ONE barrier, three dependent twists in registers, store + temper + stream the
// three outputs, ONE barrier -- instead of three load/barrier/store/barrier rounds.
constexpr int kMtThreads = 256;

// regenerate 624-word blocks from the block state in x[] and stream the tempered words to out[0..n): the three-phase walk above
__device__ __forceinline__ void mt_generate(uint32_t *x, long long n, uint32_t *__restrict__ out)
{
    constexpr int D = kMtN - kMtM;                   // 227
    const int t = threadIdx.x;
    const bool a1 = t < D, a3 = t + 2 * D < kMtN, last = t + 2 * D == kMtN - 1;
    for (long long base = 0; base < n; base += kMtN) {
        uint32_t v1 = 0, v2 = 0, v3 = 0;
        if (a1) {
            const uint32_t o0 = x[t], o1 = x[t + 1], om = x[t + kMtM];
            const uint32_t p0 = x[t + D], p1 = x[t + D + 1];
            v1 = om ^ mt_twist(o0, o1);
            v2 = v1 ^ mt_twist(p0, p1);
            if (a3) {
                const uint32_t q0 = x[t + 2 * D];
                uint32_t q1;
                if (last) q1 = x[kMtM] ^ mt_twist(x[0], x[1]);   // the NEW x[0], recomputed from old words
                else q1 = x[t + 2 * D + 1];
                v3 = v2 ^ mt_twist(q0, q1);
            }
        }
        __syncthreads();                             // every old word has been read
        if (a1) {
            x[t] = v1;
            x[t + D] = v2;
            if (base + t < n) out[base + t] = mt_temper(v1);
            if (base + t + D < n) out[base + t + D] = mt_temper(v2);
            if (a3) {
                x[t + 2 * D] = v3;
                if (base + t + 2 * D < n) out[base + t + 2 * D] = mt_temper(v3);
            }
        }
        __syncthreads();
    }
}

__device__ __forceinline__ void mt_init_genrand(uint32_t *x, uint32_t seed)   // sequential, 624 steps, once (thread 0)
{
    uint32_t s = seed;
    x[0] = s;
    for (int j = 1; j < kMtN; ++j) {
        s = 1812433253u * (s ^ (s >> 30)) + (uint32_t)j;
        x[j] = s;
    }
}

__global__ void __launch_bounds__(kMtThreads) mt19937_stream_kernel(uint32_t seed, long long n, uint32_t *__restrict__ out)
{
    __shared__ uint32_t x[kMtN + 1];
    if (threadIdx.x == 0) mt_init_genrand(x, seed);
    __syncthreads();
    mt_generate(x, n, out);
}

// ------------------------------------------------------------------ many CTAs, ONE stream: jump-ahead
// The one-word transition T of MT19937 is linear over GF(2) with a primitive characteristic polynomial phi of degree 19937, so
// T^J = g_J(T) with g_J(x) = x^J mod phi(x): the state J words ahead is sum_i g_i T^i s, a Horner walk of 19937 single steps and
// conditional XORs instead of J steps (Haramoto, Matsumoto, Nishimura, Panneton, L'Ecuyer 2008).  mt_jump_table.inc holds g for
// J = kMtSegBlocks * 624 * 2^m, m = 0 .. 7 (generated and checked against numpy by scripts/gen_mt_jump.py).  CTA k applies the
// levels of the set bits of k to the seeded state and then regenerates blocks [k * kMtSegBlocks, (k + 1) * kMtSegBlocks): the
// one-CTA kernel's 43 ms for 80 M words become one jump of at most popcount(k) passes (about half a millisecond each) plus
// 1 680 blocks per CTA.
#define DRB_MT_TABLE_QUAL __device__
#include "mt_jump_table.inc"
#undef DRB_MT_TABLE_QUAL
constexpr long long kMtSegWords = (long long)kMtSegBlocks * kMtN;

// x <- g(T) x for the polynomial of `level`; sv, hb: 624-word scratch.  All threads of the CTA call this.
__device__ __forceinline__ void mt_jump(uint32_t *x, uint32_t *sv, uint32_t *hb, int level)
{
    const int t = threadIdx.x;
    const unsigned long long *g = kMtJumpPoly[level];
    __shared__ int s_top;
    for (int j = t; j < kMtN; j += kMtThreads) { sv[j] = x[j]; hb[j] = x[j]; }      // the leading coefficient is 1: h = s
    if (t == 0) {
        int top = -1;
        for (int wd = kMtPolyWords - 1; wd >= 0 && top < 0; --wd)
            if (g[wd]) top = wd * 64 + 63 - __clzll((long long)g[wd]);
        s_top = top;
    }
    __syncthreads();
    const int top = s_top;
    int p = 0;                                       // head of the circular buffer hb (logical word j at hb[(p + j) % 624])
    unsigned long long word = 0;
    for (int i = top - 1; i >= 0; --i) {
        if ((i & 63) == 63 || i == top - 1) word = g[i >> 6];
        if (t == 0) {                                // h <- T h: one word leaves at the head, the new one takes its slot
            const int p1 = p + 1 < kMtN ? p + 1 : p + 1 - kMtN, pm = p + kMtM < kMtN ? p + kMtM : p + kMtM - kMtN;
            hb[p] = hb[pm] ^ mt_twist(hb[p], hb[p1]);
        }
        p = p + 1 < kMtN ? p + 1 : 0;
        if ((word >> (i & 63)) & 1ull) {             // uniform across the CTA: h <- h + s
            __syncthreads();
            for (int j = t; j < kMtN; j += kMtThreads) {
                const int q = p + j < kMtN ? p + j : p + j - kMtN;
                hb[q] ^= sv[j];
            }
            __syncthreads();
        }
    }
    __syncthreads();
    for (int j = t; j < kMtN; j += kMtThreads) {
        const int q = p + j < kMtN ? p + j : p + j - kMtN;
        x[j] = hb[q];
    }
    __syncthreads();
}

// CTA k: words [k * kMtSegWords, min(n, (k + 1) * kMtSegWords)) of the stream of `seed`
__global__ void __launch_bounds__(kMtThreads) mt19937_segments_kernel(uint32_t seed, long long n, uint32_t *__restrict__ out)
{
    __shared__ uint32_t x[kMtN + 1], sv[kMtN], hb[kMtN];
    const long long k = blockIdx.x, first = k * kMtSegWords;
    if (first >= n) return;
    if (threadIdx.x == 0) mt_init_genrand(x, seed);
    __syncthreads();
    for (int level = 0; level < kMtJumpLevels; ++level)
        if ((k >> level) & 1) mt_jump(x, sv, hb, level);
    const long long cnt = n - first < kMtSegWords ? n - first : kMtSegWords;
    mt_generate(x, cnt, out + first);
}

// one-off device check of the jump table and kernel: CTA m verifies g_{m+1}(T) s == g_m(T) g_m(T) s (levels chain up from
// level 0, which the host compares against the sequential kernel); ok[m] = 1 when equal in all 19 937 state bits
__global__ void __launch_bounds__(kMtThreads) mt19937_jump_check_kernel(uint32_t seed, int *__restrict__ ok)
{
    __shared__ uint32_t a[kMtN + 1], b[kMtN + 1], sv[kMtN], hb[kMtN];
    __shared__ int s_bad;
    const int m = blockIdx.x;
    if (threadIdx.x == 0) { mt_init_genrand(a, seed + 17u * (uint32_t)m); s_bad = 0; }
    __syncthreads();
    for (int j = threadIdx.x; j < kMtN; j += kMtThreads) b[j] = a[j];
    __syncthreads();
    mt_jump(a, sv, hb, m + 1);
    mt_jump(b, sv, hb, m);
    mt_jump(b, sv, hb, m);
    for (int j = threadIdx.x; j < kMtN; j += kMtThreads) {
        const uint32_t d = (a[j] ^ b[j]) & (j == 0 ? 0x80000000u : 0xffffffffu);   // word 0 of a block state: only its top bit lives on
        if (d) atomicExch(&s_bad, 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) ok[m] = s_bad ? 0 : 1;
}

struct FyParams {
    long long n;
    const uint32_t *w;           // MT19937 outputs, one per iteration
    long long *a;                // the permutation (int64, what torch.randperm returns)
    unsigned long long *r;       // reservation cells
    uint32_t *fail[2];           // unfinished iterations carried into the next round
    unsigned *cnt;               // [2] fail counters, [2] = rounds run (diagnostic)
    unsigned long long *barrier;
    long long cap;               // capacity of each fail list
};

constexpr int kFyThreads = 256;
constexpr long long kFyMinWindow = 4096;

__global__ void __launch_bounds__(kFyThreads) fisher_yates_kernel(FyParams p)
{
    const long long gtid = (long long)blockIdx.x * kFyThreads + threadIdx.x;
    const long long gsz = (long long)gridDim.x * kFyThreads;
    const int lane = threadIdx.x & 31;
    const long long n = p.n;
    unsigned long long epoch = 0;
    for (long long k = gtid; k < n; k += gsz) {
        p.a[k] = k;
        p.r[k] = ~0ull;
    }
    grid_barrier(p.barrier, epoch);
    long long s = 0;             // next fresh iteration
    long long f = 0;             // failed iterations waiting in fail[cur]
    unsigned round = 0;
    int cur = 0;
    while (s < n - 1 || f > 0) {
        long long m = n - 1 - s;
        const long long want = max(kFyMinWindow, (n - s) >> 3);
        if (m > want) m = want;
        if (m > p.cap - f) m = p.cap - f;            // the next fail list must be able to hold this round's iterations
        const long long total = f + m;
        const uint32_t *fc = p.fail[cur];
        uint32_t *fn = p.fail[cur ^ 1];
        const unsigned long long hi = (unsigned long long)(~round) << 32;   // newer rounds win the atomicMin
        // ---- reserve: both cells of every candidate iteration receive min(iteration index)
        for (long long e = gtid; e < total; e += gsz) {
            const long long i = e < f ? (long long)__ldcg(fc + e) : s + (e - f);
            const long long h = i + (long long)(__ldg(p.w + i) % (uint32_t)(n - i));
            const unsigned long long key = hi | (unsigned long long)i;
            atomicMin(p.r + i, key);
            if (h != i) atomicMin(p.r + h, key);
        }
        grid_barrier(p.barrier, epoch);
        // ---- commit: owners of both cells swap; the others queue for the next round
        const long long rounds_e = (total + gsz - 1) / gsz;
        for (long long q = 0; q < rounds_e; ++q) {
            const long long e = q * gsz + gtid;
            bool failed = false;
            long long i = 0;
            if (e < total) {
                i = e < f ? (long long)__ldcg(fc + e) : s + (e - f);
                const long long h = i + (long long)(__ldg(p.w + i) % (uint32_t)(n - i));
                const unsigned long long key = hi | (unsigned long long)i;
                const bool ok = __ldcg(p.r + i) == key && __ldcg(p.r + h) == key;
                if (ok) {
                    if (h != i) {
                        const long long ai = __ldcg(p.a + i), ah = __ldcg(p.a + h);
                        __stcg(p.a + i, ah);
                        __stcg(p.a + h, ai);
                    }
                } else {
                    failed = true;
                }
            }
            const unsigned ballot = __ballot_sync(0xffffffffu, failed);
            if (ballot) {
                unsigned base = 0;
                if (lane == 0) base = atomicAdd(p.cnt + (cur ^ 1), (unsigned)__popc(ballot));
                base = __shfl_sync(0xffffffffu, base, 0);
                if (failed) fn[base + __popc(ballot & ((1u << lane) - 1u))] = (uint32_t)i;
            }
        }
        grid_barrier(p.barrier, epoch);
        f = (long long)__ldcg(p.cnt + (cur ^ 1));
        if (gtid == 0) p.cnt[cur] = 0u;              // everyone read it one round ago; next written after the next barrier
        s += m;
        ++round;
        cur ^= 1;
    }
    if (gtid == 0) p.cnt[2] = round;
}

static inline size_t rp_align(size_t x) { return (x + 255) & ~(size_t)255; }

struct RpLayout {
    size_t w, r, f0, f1, hdr, total;
    long long cap;
};
static RpLayout rp_layout(long long n)
{
    RpLayout L;
    L.cap = n / 2 + 2 * kFyMinWindow;
    size_t off = 0;
    L.hdr = off; off += 256;
    L.w = off;   off += rp_align(sizeof(uint32_t) * (size_t)(n > 0 ? n : 1));
    L.r = off;   off += rp_align(sizeof(unsigned long long) * (size_t)(n > 0 ? n : 1));
    L.f0 = off;  off += rp_align(sizeof(uint32_t) * (size_t)L.cap);
    L.f1 = off;  off += rp_align(sizeof(uint32_t) * (size_t)L.cap);
    L.total = off;
    return L;
}

}  // namespace drb

using namespace drb;

extern "C" size_t drb_randperm_workspace_bytes(int64_t n) { return rp_layout(n).total; }

// The segmented kernel is used only after a one-off check on this device (per process): (1) the words of the first four
// segments equal the sequential kernel's, (2) every higher jump level equals two applications of the level below.  Otherwise
// the one-CTA kernel keeps running (a line on stderr says so).
static bool mt_segments_verified()
{
    static const bool no_par = getenv("DRB_MT_SEQUENTIAL") != nullptr;   // developer switch
    if (no_par) return false;
    static std::mutex mu;
    static int state = -1;
    std::lock_guard<std::mutex> lock(mu);
    if (state >= 0) return state == 1;
    state = 0;
    const long long n = 3 * kMtSegWords + 1234;
    uint32_t *da = nullptr, *db = nullptr;
    int *dok = nullptr;
    bool good = cudaMalloc(&da, n * 4) == cudaSuccess && cudaMalloc(&db, n * 4) == cudaSuccess &&
                cudaMalloc(&dok, sizeof(int) * kMtJumpLevels) == cudaSuccess;
    if (good) {
        const uint32_t seed = 20240229u;
        mt19937_stream_kernel<<<1, kMtThreads, 0, (cudaStream_t)0>>>(seed, n, da);
        mt19937_segments_kernel<<<4, kMtThreads, 0, (cudaStream_t)0>>>(seed, n, db);
        mt19937_jump_check_kernel<<<kMtJumpLevels - 1, kMtThreads, 0, (cudaStream_t)0>>>(seed, dok);
        std::vector<uint32_t> ha((size_t)n), hb((size_t)n);
        int hok[kMtJumpLevels] = {0};
        good = cudaMemcpy(ha.data(), da, n * 4, cudaMemcpyDeviceToHost) == cudaSuccess &&
               cudaMemcpy(hb.data(), db, n * 4, cudaMemcpyDeviceToHost) == cudaSuccess &&
               cudaMemcpy(hok, dok, sizeof(int) * (kMtJumpLevels - 1), cudaMemcpyDeviceToHost) == cudaSuccess;
        good = good && memcmp(ha.data(), hb.data(), (size_t)n * 4) == 0;
        for (int m = 0; m < kMtJumpLevels - 1; ++m) good = good && hok[m] == 1;
    }
    cudaFree(da); cudaFree(db); cudaFree(dok);
    cudaGetLastError();
    if (good) state = 1;
    else fprintf(stderr, "[daisyrec_b200] segmented MT19937 kernel did not reproduce the sequential stream: using the one-CTA kernel\n");
    return state == 1;
}

// d_mt_words[0..n) = first n 32-bit outputs of MT19937 seeded like at::mt19937(seed) / numpy.random.seed(seed & 0xffffffff)
extern "C" int drb_mt19937_stream(uint64_t seed, int64_t n, uint32_t *d_out, void *stream)
{
    DRB_REQUIRE(d_out && n >= 0, "mt19937_stream: bad arguments");
    if (n == 0) return DRB_OK;
    const long long segs = (n + kMtSegWords - 1) / kMtSegWords;
    if (segs >= 2 && segs <= (1ll << kMtJumpLevels) && mt_segments_verified())
        mt19937_segments_kernel<<<(int)segs, kMtThreads, 0, (cudaStream_t)stream>>>((uint32_t)(seed & 0xffffffffull), n, d_out);
    else
        mt19937_stream_kernel<<<1, kMtThreads, 0, (cudaStream_t)stream>>>((uint32_t)(seed & 0xffffffffull), n, d_out);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}

// which kernel drb_mt19937_stream runs for n words: 1 = segmented (after its one-off device check), 0 = one CTA
extern "C" int drb_mt19937_stream_variant(int64_t n)
{
    const long long segs = (n + kMtSegWords - 1) / kMtSegWords;
    return (segs >= 2 && segs <= (1ll << kMtJumpLevels) && mt_segments_verified()) ? 1 : 0;
}

// d_perm[0..n) = torch.randperm(n, generator=G) for a CPU generator G with G.manual_seed(seed), computed on the device.
extern "C" int drb_randperm_torch(uint64_t seed, int64_t n, int64_t *d_perm, void *d_ws, void *stream)
{
    DRB_REQUIRE(d_perm && d_ws && n >= 0, "randperm_torch: bad arguments");
    DRB_REQUIRE(n < (int64_t)(0xffffffffull / 20), "randperm_torch: n=%lld is beyond ATen's Fisher-Yates branch (n < 2^32/20)",
                (long long)n);
    if (n == 0) return DRB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    RpLayout L = rp_layout(n);
    char *ws = (char *)d_ws;
    DRB_CUDA(cudaMemsetAsync(ws + L.hdr, 0, 256, st));
    int rc = drb_mt19937_stream(seed, n, (uint32_t *)(ws + L.w), stream);
    if (rc != DRB_OK) return rc;
    FyParams p;
    p.n = n;
    p.w = (const uint32_t *)(ws + L.w);
    p.a = (long long *)d_perm;
    p.r = (unsigned long long *)(ws + L.r);
    p.fail[0] = (uint32_t *)(ws + L.f0);
    p.fail[1] = (uint32_t *)(ws + L.f1);
    p.barrier = (unsigned long long *)(ws + L.hdr);
    p.cnt = (unsigned *)(ws + L.hdr + 64);
    p.cap = L.cap;
    static thread_local int per_sm = 0;
    if (!per_sm) DRB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fisher_yates_kernel, kFyThreads, 0));
    DRB_REQUIRE(per_sm > 0, "fisher_yates_kernel does not fit on an SM");
    long long want = (n + kFyThreads * 4 - 1) / (kFyThreads * 4);
    long long max_grid = (long long)per_sm * sm_count();
    int grid = (int)(want < 1 ? 1 : (want > max_grid ? max_grid : want));
    void *args[] = {&p};
    DRB_CUDA(cudaLaunchCooperativeKernel((void *)fisher_yates_kernel, dim3(grid), dim3(kFyThreads), args, 0, st));
    return DRB_OK;
}
