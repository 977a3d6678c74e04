// spmm.cuh -- the segmented-CSR sparse x dense product of lightgcn.cu, shared with ngcf.cu.
#pragma once
#include "common.cuh"

namespace drb {

struct Adj {
    const int64_t *row_ptr;
    const int32_t *col;
    const float *val;
    const int32_t *seg_row;      // row of every <= 256-edge segment (drb_lgcn_segments)
    const int64_t *seg_ptr;
    long long nseg, n;
};

// Y = A X  ([n, F] fp32, row-major);  S != nullptr: S += A X as well (LightGCN's layer sum)
int launch_spmm(const Adj &a, const float *X, float *Y, float *S, int F, cudaStream_t st);

// Node dropout of NGCF (the reference's SparseDropout): every stored entry of A is kept independently, keyed by
// (seed, forward counter, CSR slot) through the common keep rule -- a kept entry weighs val * inv_keep (fp32), a dropped one
// nothing.  mirror == nullptr: Y = A_drop X.  mirror[e] = the slot of (c, r) for the slot e = (r, c): Y = A_drop^T X over the
// same CSR (A structurally symmetric with symmetric values, so only the keep is read at the mirror slot).
constexpr uint32_t kEdgeDropDomain = 0x80000000u;   // counter word 2 of the edge masks (the message masks put a layer there)
struct EdgeDrop {
    const int32_t *mirror;
    uint32_t k0, k1, fwd, thresh;
    float inv_keep;
};
int launch_spmm_drop(const Adj &a, const float *X, float *Y, int F, const EdgeDrop &ed, cudaStream_t st);

#ifdef __CUDACC__
// the four Philox words of CSR slots 4 * chunk .. 4 * chunk + 3
__device__ __forceinline__ void edge_words(const EdgeDrop &d, unsigned long long chunk, uint32_t (&c)[4])
{
    c[0] = (uint32_t)chunk; c[1] = (uint32_t)(chunk >> 32); c[2] = kEdgeDropDomain; c[3] = d.fwd;
    philox4x32(c, d.k0, d.k1);
}
#endif

}  // namespace drb
