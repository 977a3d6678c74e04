// gemm.cuh -- plain entry points of the dense-layer helpers in neumf.cu: the GEMM dispatcher (dtype 0: fp32 CUDA cores,
// 1: bf16 wgmma), bias-gradient column sums and the optimiser step on a flat parameter block.
#pragma once
#include "common.cuh"

namespace drb {

struct WsHeader;

// C[M,N] = A[M,K] B[N,K]^T        (Linear forward: activations x weight^T)
int gemm_nt(int dtype, long long M, int N, int K, const float *A, long long lda, const float *B, long long ldb, float *C,
            long long ldc, cudaStream_t st);
// C[M,N] = A[M,K] B[K,N]          (input gradient: dZ x weight)
int gemm_nn(int dtype, long long M, int N, int K, const float *A, long long lda, const float *B, long long ldb, float *C,
            long long ldc, cudaStream_t st);
// C[N,M] += (A[K,M]^T B[K,N])^T   (weight gradient [out, in] += dZ^T X, computed with the wide dimension on the MMA rows; split-K)
int gemm_tn_acc_t(int dtype, long long M, int N, int K, const float *A, long long lda, const float *B, long long ldb, float *C,
                  long long ldc, cudaStream_t st);
// C[M,N] = A[K,M]^T B[K,N]        (weight gradient written, not accumulated: fp32, each output summed over k in order)
int gemm_tn(long long M, int N, int K, const float *A, long long lda, const float *B, long long ldb, float *C, long long ldc,
            cudaStream_t st);
// C + z (M ldc) = A[M, Kz] B[Kz, N] for the z-th of `slices` equal k ranges (fp32; the caller sums the slices in a fixed order)
int gemm_nn_slices(long long M, int N, int K, const float *A, long long lda, const float *B, long long ldb, float *C,
                   long long ldc, int slices, cudaStream_t st);
// gb[n] += sum_m dZ[m, n]          (bias gradient, N <= 256)
int colsum_acc(const float *dZ, long long M, int N, float *gb, cudaStream_t st);
// the same over the 2B rows of a pairwise step, each pos row m added to its neg row B + m first
int colsum_pairs_acc(const float *dZ, long long B, int N, float *gb, cudaStream_t st);
// optimiser step of h on the flat block W[n] with gradient g (SGD, or torch.optim.Adam's single-tensor rule with state m, v at
// step adam_step0 + 1); clears g.  Does nothing once hdr->status is set (a NaN loss).
int dense_update(float *W, float *g, float *m, float *v, long long n, const drb_hyper *h, long long adam_step0,
                 const WsHeader *hdr, cudaStream_t st);

}  // namespace drb
