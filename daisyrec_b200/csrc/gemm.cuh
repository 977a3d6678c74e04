// gemm.cuh -- plain entry points of the dense-layer GEMM dispatcher in neumf.cu (dtype 0: fp32 CUDA cores, 1: bf16 wgmma).
#pragma once
#include "common.cuh"

namespace drb {

// C[M,N] = A[M,K] B[N,K]^T        (Linear forward: activations x weight^T)
int gemm_nt(int dtype, long long M, int N, int K, const float *A, long long lda, const float *B, long long ldb, float *C,
            long long ldc, cudaStream_t st);
// C[M,N] = A[M,K] B[K,N]          (input gradient: dZ x weight)
int gemm_nn(int dtype, long long M, int N, int K, const float *A, long long lda, const float *B, long long ldb, float *C,
            long long ldc, cudaStream_t st);
// C[N,M] += (A[K,M]^T B[K,N])^T   (weight gradient [out, in] += dZ^T X, computed with the wide dimension on the MMA rows; split-K)
int gemm_tn_acc_t(int dtype, long long M, int N, int K, const float *A, long long lda, const float *B, long long ldb, float *C,
                  long long ldc, cudaStream_t st);
// gb[n] += sum_m dZ[m, n]          (bias gradient, N <= 256)
int colsum_acc(const float *dZ, long long M, int N, float *gb, cudaStream_t st);
// the same over the 2B rows of a pairwise step, each pos row m added to its neg row B + m first
int colsum_pairs_acc(const float *dZ, long long B, int N, float *gb, cudaStream_t st);

}  // namespace drb
