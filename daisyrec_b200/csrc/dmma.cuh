// dmma.cuh -- fp64 tensor-core (DMMA, mma.sync m8n8k4 .f64) tile product for sm_90a.
//
// dmma_nt_64 accumulates acc += A[64 x K] * B[64 x K]^T for one 256-thread CTA: A and B are row-major with K contiguous
// (both operands are "rows of items"), staged through shared memory 32 columns at a time.  Warp w owns rows
// 32 (w >> 2) .. +32 and columns 16 (w & 3) .. +16 of the tile: 4 x 2 fragments of 8 x 8.  Fragment (mi, ni) holds
// C[32 (w >> 2) + 8 mi + g][16 (w & 3) + 8 ni + 2 t + {0, 1}], g = lane / 4, t = lane % 4 (PTX m8n8k4 f64 layout).
// Every product of two doubles is rounded once and summed in a fixed order, so a tile is bitwise reproducible.
#pragma once
#include "common.cuh"

namespace drb {

constexpr int kDmmaTile = 64;
constexpr int kDmmaK = 32;

struct DmmaSmem {
    double a[kDmmaTile][kDmmaK + 4];   // +4 doubles per row: the 8 rows of a fragment land in distinct bank pairs
    double b[kDmmaTile][kDmmaK + 4];
};

__device__ __forceinline__ void dmma_m8n8k4(double (&d)[2], double a, double b)
{
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
                 : "+d"(d[0]), "+d"(d[1])
                 : "d"(a), "d"(b));
}

// lda, ldb even and K a multiple of kDmmaK; all 64 rows of A and B must be readable (callers pad their buffers).
__device__ __forceinline__ void dmma_nt_64(const double *__restrict__ A, long long lda, const double *__restrict__ B,
                                           long long ldb, int K, double (&acc)[4][2][2], DmmaSmem &sm)
{
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int wm = (warp >> 2) * 32, wn = (warp & 3) * 16;
    for (int k0 = 0; k0 < K; k0 += kDmmaK) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int idx = tid + q * 256, row = idx >> 4, c2 = (idx & 15) * 2;
            *reinterpret_cast<double2 *>(&sm.a[row][c2]) = __ldcg(reinterpret_cast<const double2 *>(A + row * lda + k0 + c2));
            *reinterpret_cast<double2 *>(&sm.b[row][c2]) = __ldcg(reinterpret_cast<const double2 *>(B + row * ldb + k0 + c2));
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < kDmmaK; kk += 4) {
            double a[4], b[2];
#pragma unroll
            for (int mi = 0; mi < 4; ++mi) a[mi] = sm.a[wm + mi * 8 + g][kk + t];
#pragma unroll
            for (int ni = 0; ni < 2; ++ni) b[ni] = sm.b[wn + ni * 8 + g][kk + t];
#pragma unroll
            for (int mi = 0; mi < 4; ++mi)
#pragma unroll
                for (int ni = 0; ni < 2; ++ni) dmma_m8n8k4(acc[mi][ni], a[mi], b[ni]);
        }
        __syncthreads();
    }
}

// (row, col) inside the 64 x 64 tile of element e of fragment (mi, ni) of this thread
__device__ __forceinline__ int dmma_row(int mi)
{
    return ((threadIdx.x >> 5) >> 2) * 32 + mi * 8 + ((threadIdx.x & 31) >> 2);
}
__device__ __forceinline__ int dmma_col(int ni, int e)
{
    return ((threadIdx.x >> 5) & 3) * 16 + ni * 8 + (threadIdx.x & 3) * 2 + e;
}

}  // namespace drb
