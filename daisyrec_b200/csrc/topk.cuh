// topk.cuh -- the block-wide top-k of fp64 scores that the rank / full_rank kernels of ease.cu and itemknn.cu share.
#pragma once
#include "common.cuh"

namespace drb {

// 64-bit key ordered as the fp64 score (-0 counted as +0)
__device__ __forceinline__ unsigned long long score_key(double s)
{
    if (s == 0.0) s = 0.0;
    const unsigned long long b = (unsigned long long)__double_as_longlong(s);
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}

__device__ __forceinline__ bool key_before(unsigned long long ka, int pa, unsigned long long kb, int pb)
{
    return ka > kb || (ka == kb && pa < pb);
}

// top-k of sc[0 .. C) by (score descending, position ascending): k rounds of a block arg-max over the elements after the
// previous pick.  out[r] = ids ? ids[pos] : pos.
static __device__ void block_topk(const double *sc, int C, int k, const int64_t *ids, int64_t *out)
{
    __shared__ unsigned long long wk[32];
    __shared__ int wp[32];
    __shared__ unsigned long long s_lk;
    __shared__ int s_lp;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = (blockDim.x + 31) >> 5;
    unsigned long long lk = ~0ull;
    int lp = -1;
    for (int r = 0; r < k; ++r) {
        unsigned long long bk = 0;
        int bp = 0x7fffffff;
        for (int c = tid; c < C; c += blockDim.x) {
            const unsigned long long kc = score_key(sc[c]);
            if (key_before(lk, lp, kc, c) && key_before(kc, c, bk, bp)) { bk = kc; bp = c; }
        }
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) {
            const unsigned long long ok = __shfl_xor_sync(0xffffffffu, bk, off);
            const int op = __shfl_xor_sync(0xffffffffu, bp, off);
            if (key_before(ok, op, bk, bp)) { bk = ok; bp = op; }
        }
        if (lane == 0) { wk[warp] = bk; wp[warp] = bp; }
        __syncthreads();
        if (warp == 0) {
            bk = lane < nw ? wk[lane] : 0ull;
            bp = lane < nw ? wp[lane] : 0x7fffffff;
#pragma unroll
            for (int off = 16; off >= 1; off >>= 1) {
                const unsigned long long ok = __shfl_xor_sync(0xffffffffu, bk, off);
                const int op = __shfl_xor_sync(0xffffffffu, bp, off);
                if (key_before(ok, op, bk, bp)) { bk = ok; bp = op; }
            }
            if (lane == 0) {
                s_lk = bk;
                s_lp = bp;
                out[r] = ids ? ids[bp] : (int64_t)bp;
            }
        }
        __syncthreads();
        lk = s_lk;
        lp = s_lp;
        __syncthreads();
    }
}

}  // namespace drb
