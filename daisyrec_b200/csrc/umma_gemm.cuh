// umma_gemm.cuh -- bf16 tensor-core GEMM for the NeuMF tower on sm_90a: wgmma with fp32 accumulators in registers.
//
//   C[M,N] (op)= opA(A)[M,K] * opB(B)[K,N]       A, B, C fp32 in global memory; operands are rounded to bf16
//   while they are staged into shared memory, products accumulate in fp32 in the registers of the issuing warpgroup.
//
// Same call signature and epilogues as the fp32 CUDA-core sgemm_kernel in neumf.cu, so the three GEMM call sites of
// the tower (forward NT + bias + ReLU, input-gradient NN + ReLU mask, weight-gradient TN split-K) switch by dtype.
//
// One CTA (two warpgroups, 256 threads) owns a 128-row tile of C and NT >= N columns (NT in {32, 64, 128, 256}):
//   * per 32-deep K chunk all threads stage A[128x32] and B[NT x 32] into shared memory in the canonical
//     no-swizzle core-matrix layouts (8 x 16-byte core matrices; K-major for operands that are contiguous along K,
//     MN-major for the transposed operands of the backward GEMMs; LBO / SBO padded so the 16-byte staging stores are
//     bank-conflict free), fence.proxy.async, then warpgroup g issues wgmma.m64n32k16 over rows [64g, 64g + 64) for
//     every 32-column slice of B and waits for its own group;
//   * epilogue: each thread owns two rows x NT/4 columns of the accumulator fragment and writes them with bias / ReLU /
//     mask fused, or atomically accumulates (optionally transposed) for the split-K weight gradient.
// The tower GEMMs are skinny (N, K <= 128 against M ~ 10^6): they are bound by streaming A from HBM, not by the
// tensor pipe, so the kernel relies on several resident CTAs per SM for overlap rather than on an intra-CTA pipeline.
#pragma once
#include <cuda_bf16.h>

#include "common.cuh"

namespace drb {

constexpr int kUmmaBK = 32;        // K elements staged per chunk (2 MMAs of K=16)
constexpr int kUmmaMaxN = 256;
constexpr int kUmmaThreads = 256;  // two warpgroups, 64 tile rows each

// wgmma shared-memory matrix descriptor, no swizzle: start [0,14) >>4, LBO [16,30) >>4, SBO [32,46) >>4,
// base_offset [49,52) = 0, layout_type [62,64) = 0 (interleave).  LBO is the stride between core matrices along K,
// SBO the stride between core matrices along M / N, for K-major and MN-major operands alike.
__device__ __forceinline__ uint64_t umma_smem_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes)
{
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3fffu);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3fffu) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3fffu) << 32;
    return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// keeps the compiler from moving accesses of an accumulator across the asynchronous MMA that owns it
template <int N>
__device__ __forceinline__ void wgmma_fence_operand(float (&d)[N])
{
#pragma unroll
    for (int e = 0; e < N; ++e) asm volatile("" : "+f"(d[e])::"memory");
}

// D[64 x 32] (+)= A[64 x 16] * B[16 x 32], bf16 operands from shared memory, fp32 accumulators.  TA / TB: 0 = K-major,
// 1 = MN-major operand image.  Fragment: d[4 nb + 2 i + c] = D(16 warp + lane / 4 + 8 i, 8 nb + 2 (lane % 4) + c).
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n32(float (&d)[16], uint64_t da, uint64_t db, uint32_t accumulate)
{
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
}
// the same with 16 columns: d[4 nb + 2 i + c], nb in {0, 1}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n16(float (&d)[8], uint64_t da, uint64_t db, uint32_t accumulate)
{
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %11, %12;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
}

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b)
{
    __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t *>(&v);
}

// Operand tiles in shared memory (no swizzle, 8 x 16-byte core matrices), padded so that the 16-byte staging stores of a
// quarter warp fall into distinct bank groups:
//   K-major  (source contiguous along K):   elem(r, k) at (k/8)*LBO + (r/8)*128 + (r%8)*16 + (k%8)*2,  LBO = rows/8*128 + 32, SBO = 128
//   MN-major (source contiguous along rows): elem(r, k) at (k/8)*LBO + (r/8)*144 + (k%8)*16 + (r%8)*2,  LBO = rows/8*144,      SBO = 144
// Either way one work item converts 8 consecutive source floats to bf16 and issues ONE 16-byte shared store.
__host__ __device__ __forceinline__ uint32_t umma_lbo(bool mn_major, int rows)
{
    return mn_major ? (uint32_t)(rows / 8) * 144u : (uint32_t)(rows / 8) * 128u + 32u;
}
__host__ __device__ __forceinline__ uint32_t umma_sbo(bool mn_major) { return mn_major ? 144u : 128u; }

//   MN = false: src(r, k) = S[(r0 + r) * ld + k]       MN = true: src(r, k) = S[k * ld + (r0 + r)]
// An item reads its 8 floats with two 16-byte loads only when that address is 16-byte aligned: S itself aligned, ld a multiple
// of 4, and the item's start a multiple of 4 (k always is: chunks start at multiples of kUmmaBK; the row is checked).  Column
// slices of a wider matrix (NGCF's T half of [S | T] at an input width that is not a multiple of 4, its W1 / W2 blocks at a
// float offset in the parameter block that is not a multiple of 4 -- W2 starts out * (in + 1) floats after W1, odd for an
// odd out and an even in) are staged float by float.
template <bool MN>
__device__ __forceinline__ void umma_stage_tile(unsigned char *smem, int rows, const float *__restrict__ S, long long ld,
                                                long long r0, long long r_lim, int k0, int k_lim, int tid, int nthreads)
{
    const uint32_t lbo = umma_lbo(MN, rows);
    const int items = MN ? (rows / 8) * kUmmaBK : rows * (kUmmaBK / 8);
    const bool vec = ((reinterpret_cast<uintptr_t>(S) & 15) == 0) && ((ld & 3) == 0);
    for (int it = tid; it < items; it += nthreads) {
        float v[8];
        uint32_t off;
        if (!MN) {
            const int r = it / (kUmmaBK / 8), c1 = it % (kUmmaBK / 8);    // 4 lanes read 128 contiguous bytes of a row
            const long long gr = r0 + r;
            const int k = k0 + c1 * 8;
            if (vec && gr < r_lim && k + 8 <= k_lim) {
                const float4 *p = reinterpret_cast<const float4 *>(S + gr * ld + k);
                float4 a = __ldg(p), b = __ldg(p + 1);
                v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
            } else {
#pragma unroll
                for (int e = 0; e < 8; ++e) v[e] = (gr < r_lim && k + e < k_lim) ? __ldg(S + gr * ld + k + e) : 0.f;
            }
            off = (uint32_t)c1 * lbo + (uint32_t)(r / 8) * 128u + (uint32_t)(r % 8) * 16u;
        } else {
            const int rg = it % (rows / 8), c = it / (rows / 8);          // consecutive lanes read consecutive row groups
            const long long gr = r0 + (long long)rg * 8;
            const int k = k0 + c;
            if (vec && k < k_lim && gr + 8 <= r_lim && ((gr & 3) == 0)) {
                const float4 *p = reinterpret_cast<const float4 *>(S + (long long)k * ld + gr);
                float4 a = __ldg(p), b = __ldg(p + 1);
                v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
            } else {
#pragma unroll
                for (int e = 0; e < 8; ++e) v[e] = (k < k_lim && gr + e < r_lim) ? __ldg(S + (long long)k * ld + gr + e) : 0.f;
            }
            off = (uint32_t)(c / 8) * lbo + (uint32_t)rg * 144u + (uint32_t)(c % 8) * 16u;
        }
        uint4 o;
        o.x = pack_bf16x2(v[0], v[1]); o.y = pack_bf16x2(v[2], v[3]);
        o.z = pack_bf16x2(v[4], v[5]); o.w = pack_bf16x2(v[6], v[7]);
        *reinterpret_cast<uint4 *>(smem + off) = o;
    }
}

// EPI 0: C = acc   1: C = relu(acc + bias[n])   2: C = acc * (ref(m,n) > 0)   3: atomicAdd(C, acc) (split-K over grid.z)
// EPI 4: atomicAdd(C^T, acc) -- transposed accumulate C[n*ldc + m] (split-K)
template <bool TA, bool TB, int EPI, int NT>
__global__ void __launch_bounds__(kUmmaThreads) umma_gemm_kernel(int M, int N, int K, const float *__restrict__ A, long long lda,
                                                                 const float *__restrict__ B, long long ldb, float *__restrict__ C,
                                                                 long long ldc, const float *__restrict__ bias,
                                                                 const float *__restrict__ ref, long long ldref, int k_chunk,
                                                                 float alpha)
{
    constexpr int kABytes = (kUmmaBK / 8) * (128 / 8) * 144;                 // worst case (MN-major) A tile
    constexpr int kBBytes = (kUmmaBK / 8) * (NT / 8) * 144;
    constexpr int NS = NT / 32;                                               // 32-column slices per warpgroup
    __shared__ __align__(128) unsigned char s_all[kABytes + kBBytes];
    unsigned char *sA = s_all, *sB = s_all + kABytes;
    // A(m,k) = A[k*lda + m] (TA) and B(k,n) = B[k*ldb + n] (!TB) are contiguous along the MN dimension -> MN-major tiles
    constexpr bool A_MN = TA, B_MN = !TB;
    const int tid = threadIdx.x, wg = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31;
    const long long m0 = (long long)blockIdx.x * 128;
    const int kb = (EPI >= 3) ? blockIdx.z * k_chunk : 0;
    const int ke = (EPI >= 3) ? min(K, kb + k_chunk) : K;

    float acc[NS][16];
#pragma unroll
    for (int s = 0; s < NS; ++s)
#pragma unroll
        for (int e = 0; e < 16; ++e) acc[s][e] = 0.f;
    const uint32_t lboA = umma_lbo(A_MN, 128), lboB = umma_lbo(B_MN, NT);
    const uint32_t sboA = umma_sbo(A_MN), sboB = umma_sbo(B_MN);
    const uint32_t aBase = smem_u32(sA) + (uint32_t)wg * 8u * sboA, bBase = smem_u32(sB);   // this warpgroup's 64 rows
    for (int k0 = kb; k0 < ke; k0 += kUmmaBK) {
        umma_stage_tile<A_MN>(sA, 128, A, lda, m0, M, k0, ke, tid, kUmmaThreads);
        umma_stage_tile<B_MN>(sB, NT, B, ldb, 0, N, k0, ke, tid, kUmmaThreads);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy stores -> visible to the tensor core
        __syncthreads();
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < kUmmaBK / 16; ++kk) {
            const uint64_t da = umma_smem_desc(aBase + kk * 2 * lboA, lboA, sboA);
#pragma unroll
            for (int s = 0; s < NS; ++s)
                wgmma_m64n32<A_MN, B_MN>(acc[s], da, umma_smem_desc(bBase + s * 4 * sboB + kk * 2 * lboB, lboB, sboB), 1u);
        }
        wgmma_commit();
        wgmma_wait_all();
#pragma unroll
        for (int s = 0; s < NS; ++s) wgmma_fence_operand(acc[s]);
        __syncthreads();                                                 // both warpgroups done reading before restaging
    }
    if (kb >= ke) return;
    const long long mrow = m0 + wg * 64 + warp * 16 + (lane >> 2);
#pragma unroll
    for (int s = 0; s < NS; ++s) {
#pragma unroll
        for (int nb = 0; nb < 4; ++nb) {
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const long long m = mrow + 8 * i;
                if (m >= M) continue;
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const int n = s * 32 + nb * 8 + 2 * (lane & 3) + c;
                    if (n >= N) continue;
                    float v = acc[s][nb * 4 + i * 2 + c];
                    if (EPI == 1) { v += bias[n]; v = v > 0.f ? v : 0.f; }
                    if (EPI == 2) { v = (ref[m * ldref + n] > 0.f) ? v * alpha : 0.f; }
                    if (EPI == 3) atomicAdd(C + m * ldc + n, v);
                    else if (EPI == 4) atomicAdd(C + (long long)n * ldc + m, v);
                    else C[m * ldc + n] = v;
                }
            }
        }
    }
}

template <bool TA, bool TB, int EPI, int NT>
static void launch_umma_gemm_nt(dim3 grid, long long M, int N, int K, const float *A, long long lda, const float *B, long long ldb,
                                float *C, long long ldc, const float *bias, const float *ref, long long ldref, int k_chunk,
                                cudaStream_t st, float alpha)
{
    umma_gemm_kernel<TA, TB, EPI, NT><<<grid, kUmmaThreads, 0, st>>>((int)M, N, K, A, lda, B, ldb, C, ldc, bias, ref, ldref,
                                                                     k_chunk, alpha);
}

template <bool TA, bool TB, int EPI>
static int launch_umma_gemm(long long M, int N, int K, const float *A, long long lda, const float *B, long long ldb, float *C,
                            long long ldc, const float *bias, const float *ref, long long ldref, cudaStream_t st,
                            float alpha = 1.f)
{
    if (M <= 0 || N <= 0 || K <= 0) return DRB_OK;
    DRB_REQUIRE(N <= kUmmaMaxN, "umma_gemm: N=%d exceeds %d", N, kUmmaMaxN);
    dim3 grid((unsigned)((M + 127) / 128), 1, 1);
    int k_chunk = K;
    if (EPI >= 3) {   // split-K: the [out x in] result is one tile, parallelism comes from the K (row) dimension.
        // Each CTA runs its K steps back to back (stage -> mma -> wait), so latency is hidden by CTA count: aim at
        // ~8 resident CTAs per SM, but keep >= 512 rows per chunk so the atomic epilogue stays a small fraction.
        long long want = (long long)sm_count() * 8;
        long long max_chunks = (K + 511) / 512;
        long long chunks = want < max_chunks ? want : max_chunks;
        if (chunks < 1) chunks = 1;
        k_chunk = (int)(((K + chunks - 1) / chunks + kUmmaBK - 1) / kUmmaBK * kUmmaBK);
        grid.z = (unsigned)((K + k_chunk - 1) / k_chunk);
    }
    if (N <= 32) launch_umma_gemm_nt<TA, TB, EPI, 32>(grid, M, N, K, A, lda, B, ldb, C, ldc, bias, ref, ldref, k_chunk, st, alpha);
    else if (N <= 64) launch_umma_gemm_nt<TA, TB, EPI, 64>(grid, M, N, K, A, lda, B, ldb, C, ldc, bias, ref, ldref, k_chunk, st, alpha);
    else if (N <= 128) launch_umma_gemm_nt<TA, TB, EPI, 128>(grid, M, N, K, A, lda, B, ldb, C, ldc, bias, ref, ldref, k_chunk, st, alpha);
    else launch_umma_gemm_nt<TA, TB, EPI, 256>(grid, M, N, K, A, lda, B, ldb, C, ldc, bias, ref, ldref, k_chunk, st, alpha);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}

}  // namespace drb
