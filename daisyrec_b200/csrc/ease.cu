// ease.cu -- EASE (daisy/model/EASERecommender.py, Steck 2019) on the device.
//
// The reference's fit is dense linear algebra on the host: X = csr_matrix((values, (u, i))).astype(float32),
// G = X^T X + reg I (fp32 sparse product, upcast to fp64), P = np.linalg.inv(G), B = -P / diag(P) with a zero diagonal.
//
//   drb_ease_csr      values of X: each COO value summed into its slot of the sorted, duplicate-free CSR in fp64, in row
//                     order, rounded once to fp32 (scipy's duplicate sum).  Also decides whether the Gram can be exact:
//                     the smallest s in [0, 7] with every x 2^s an integer in [-127, 127] and max_i sum_u (x_ui 2^s)^2
//                     < 2^31.  By Cauchy-Schwarz that bounds every |G_ij| and every partial sum, so s8 x s8 -> s32 cannot
//                     overflow.
//   drb_ease_scale    the same decision for a CSR whose values are already in place (ItemKNN's transformed copies of X).
//   drb_ease_gram     G = X^T X + reg I, fp64 [n, n].  User chunks are expanded into a dense item-major image and the lower
//                     triangle of tiles accumulates image * image^T:
//                       exact path   s8 operands, s32 accumulation on the tensor cores (mma.sync m16n8k32), the chunk's
//                                    integer tile added to G as an exactly representable double (x 2^-2s);
//                       general path fp64 DMMA (m8n8k4) on fp64 images: fp32 x fp32 products are exact in fp64.
//                     No floating-point atomics: each tile belongs to one CTA per chunk and chunks run in order, so G is
//                     bitwise reproducible.  The exact path gives the exact Gram; it equals the reference's fp64 matrix
//                     bit for bit while max_i sum_u (x_ui 2^s)^2 < 2^24, where scipy's fp32 sums are exact as well.
//   drb_gram_image / drb_gram_panel   the same Gram by row panels, for UserKNN's [U, U] matrix that is never held whole:
//                     one dense image of the CSR's columns over all of K (s8 or fp64 as above), then G[p0 .. p0 + rows, :]
//                     on a rectangular tile grid that runs the triangle grid's tile body.  Each entry is one CTA's full-K
//                     sum, so a panel's rows do not depend on the panel size.
//   drb_ease_inverse  P = G^-1 in place by the blocked sweep operator (symmetric block Gauss-Jordan, no pivoting: G is
//                     positive definite for reg > 0).  Per pivot block k of kNb columns:
//                       D = G_kk^-1 in one CTA (scalar sweep in shared memory; a pivot <= 0 raises a sticky flag),
//                       V = column block k, W = V D (DMMA), the rank-kNb update G_ij -= W_i V_j^T on the lower tiles (DMMA),
//                       G_ik = W_i, G_kk = -D.
//                     After all blocks G holds -P in its lower triangle; it is negated and mirrored.
//   drb_ease_weights  B = -P / diag(P) by column, zero diagonal, in place.
//   drb_ease_rank     rank(): s_c = sum_i x_ui B[c, i] (the reference gathers ROWS of B for the candidates), top-K by
//                     (score descending, candidate position ascending), int64 item ids.
//   drb_ease_full_rank / drb_ease_predict   full_rank() / predict(): x_u B, streaming the rows B[i, :] of the user's items.
#include <string.h>

#include "common.cuh"
#include "dmma.cuh"
#include "topk.cuh"

namespace drb {

constexpr int kNb = 128;               // sweep pivot block
constexpr int kS8Tile = 128;           // exact Gram CTA tile
constexpr int kS8K = 64;               // its K step (bytes)
constexpr long long kImageBytes = 512ll << 20;   // budget of one user chunk's dense image

static long long round_up(long long x, long long m) { return (x + m - 1) / m * m; }

struct EaseGeom {
    long long rows;    // image rows (items, padded to the Gram tile)
    long long chunk;   // users per chunk (image columns)
    long long n128;    // rows of the sweep's panel buffers
};

static EaseGeom ease_geom(int U, int I, int scale)
{
    EaseGeom g;
    const bool exact = scale >= 0;
    g.rows = round_up(I, exact ? kS8Tile : kDmmaTile);
    long long c = kImageBytes / (g.rows * (exact ? 1 : 8)) / 64 * 64;
    const long long umax = round_up(U, 64);
    g.chunk = c < 64 ? 64 : (c > umax ? umax : c);
    g.n128 = round_up(I, kNb);
    return g;
}

struct EaseWs {
    void *image;
    double *V, *W, *D, *diag;
    int *flag;
};

static size_t carve_ease(void *base, int U, int I, int scale, EaseWs *w)
{
    const EaseGeom g = ease_geom(U, I, scale);
    size_t off = 0;
    char *b = (char *)base;
    auto take = [&](size_t bytes) {
        char *p = b ? b + off : nullptr;
        off += (bytes + 255) & ~(size_t)255;
        return p;
    };
    EaseWs t;
    t.flag = (int *)take(256);
    t.V = (double *)take(sizeof(double) * (size_t)g.n128 * kNb);
    t.W = (double *)take(sizeof(double) * (size_t)g.n128 * kNb);
    t.D = (double *)take(sizeof(double) * kNb * kNb);
    t.diag = (double *)take(sizeof(double) * (size_t)I);
    t.image = take((size_t)(g.rows * g.chunk * (scale >= 0 ? 1 : 8)));   // last: the sweep's buffers depend on I alone
    if (w) *w = t;
    return off;
}

struct CsrStats {
    unsigned smax;       // max over values of the smallest s with x 2^s integral (8: none in [0, 7])
    unsigned amax;       // max |x| as fp32 bits
    unsigned long long sqmax;   // max_i sum_u x_ui^2 as fp64 bits
};

// ---------------------------------------------------------------- X's values
// one user's stored values [b, e) folded into the statistics the exact-Gram rule reads
// (val is not __restrict__: ease_values_kernel has just written it)
__device__ __forceinline__ void row_stats(const float *val, const int32_t *__restrict__ col, long long b, long long e,
                                          double *__restrict__ colsq, CsrStats *__restrict__ st)
{
    unsigned smax = 0, amax = 0;
    for (long long k = b; k < e; ++k) {
        const float x = val[k];
        unsigned s = 8;
        if (isfinite(x)) {
            for (unsigned t = 0; t < 8; ++t) {
                const float y = ldexpf(x, (int)t);
                if (y == floorf(y)) { s = t; break; }
            }
        }
        smax = max(smax, s);
        amax = max(amax, __float_as_uint(fabsf(x)));   // NaN compares above every finite value
        atomicAdd(colsq + col[k], (double)x * (double)x);
    }
    if (e > b) {
        atomicMax(&st->smax, smax);
        atomicMax(&st->amax, amax);
    }
}

// One thread per user walks the user's COO rows in row order (d_order: stable grouping) and adds each value into its CSR
// slot: every slot's duplicates are summed in fp64 in row order, then rounded once to fp32.
__global__ void ease_values_kernel(const int64_t *__restrict__ seq_ptr, const int32_t *__restrict__ order,
                                   const int32_t *__restrict__ coo_i, const double *__restrict__ coo_v, int U,
                                   const int64_t *__restrict__ row_ptr, const int32_t *__restrict__ col,
                                   double *__restrict__ sum, float *__restrict__ val, double *__restrict__ colsq,
                                   CsrStats *__restrict__ st)
{
    for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < U; u += gridDim.x * blockDim.x) {
        const long long b = row_ptr[u], e = row_ptr[u + 1];
        for (long long k = b; k < e; ++k) sum[k] = 0.0;
        for (long long q = seq_ptr[u]; q < seq_ptr[u + 1]; ++q) {
            const int r = order[q];
            const int item = coo_i[r];
            long long lo = b, hi = e - 1;   // the item is in the row: the CSR was built from these pairs
            while (lo < hi) {
                const long long mid = (lo + hi) >> 1;
                if (col[mid] < item) lo = mid + 1; else hi = mid;
            }
            sum[lo] += coo_v[r];
        }
        for (long long k = b; k < e; ++k) val[k] = (float)sum[k];
        row_stats(val, col, b, e, colsq, st);
    }
}

// the statistics of a CSR whose values are already in place (a thread per user)
__global__ void ease_stats_kernel(const int64_t *__restrict__ row_ptr, const int32_t *__restrict__ col,
                                  const float *__restrict__ val, int U, double *__restrict__ colsq, CsrStats *__restrict__ st)
{
    for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < U; u += gridDim.x * blockDim.x)
        row_stats(val, col, row_ptr[u], row_ptr[u + 1], colsq, st);
}

__global__ void ease_sqmax_kernel(const double *__restrict__ colsq, int I, CsrStats *__restrict__ st)
{
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < I; i += gridDim.x * blockDim.x)
        atomicMax(&st->sqmax, (unsigned long long)__double_as_longlong(colsq[i]));   // non-negative: bits order as values
}

// ---------------------------------------------------------------- Gram
// image[i][u - u0] = x_ui (x 2^s as s8 on the exact path); one warp per user of the chunk.  The image is zeroed first.
template <typename T>
__global__ void ease_image_kernel(const int64_t *__restrict__ row_ptr, const int32_t *__restrict__ col,
                                  const float *__restrict__ val, int u0, int u1, long long ld, float scale, T *__restrict__ img)
{
    const int lane = threadIdx.x & 31;
    for (int u = u0 + (int)((blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5); u < u1;
         u += (int)(((long long)gridDim.x * blockDim.x) >> 5)) {
        for (long long k = row_ptr[u] + lane; k < row_ptr[u + 1]; k += 32) {
            const float x = val[k] * scale;
            T v;
            if constexpr (sizeof(T) == 1) v = (T)__float2int_rn(x); else v = (T)x;
            img[(long long)col[k] * ld + (u - u0)] = v;
        }
    }
}

// lower-triangle tile pair (bi >= bj) of linear index t
__device__ __forceinline__ void tri_pair(long long t, int &bi, int &bj)
{
    int i = (int)((sqrt(8.0 * (double)t + 1.0) - 1.0) * 0.5);
    while ((long long)i * (i + 1) / 2 > t) --i;
    while ((long long)(i + 1) * (i + 2) / 2 <= t) ++i;
    bi = i;
    bj = (int)(t - (long long)i * (i + 1) / 2);
}

__device__ __forceinline__ void imma_m16n8k32(int (&d)[4], const int (&a)[4], const int (&b)[2])
{
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
                 "{%0, %1, %2, %3};"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// Gt[r][c] += unit * (128 image rows at Ag) . (128 image rows at Bg)^T over K columns, for r < nr, c < nc (Gt: the tile's
// origin in a row-major fp64 matrix of leading dimension ldg); s8 x s8 -> s32.  8 warps as 2 x 4, each 64 x 32 of the 128 x 128
// tile: 4 x 4 fragments of m16n8k32.  One 256-thread CTA; the triangle grid below (kAdd: chunks accumulate) and the panel grid
// (a single full-K pass that stores, so the panel needs no zeroing) share it.
template <bool kAdd>
__device__ __forceinline__ void gram_s8_tile(const int8_t *__restrict__ Ag, const int8_t *__restrict__ Bg, long long ld, int K,
                                             double *__restrict__ Gt, long long ldg, int nr, int nc, double unit)
{
    __shared__ __align__(16) int8_t As[kS8Tile][kS8K + 16];   // 80-byte rows: a fragment's 8 rows hit distinct banks
    __shared__ __align__(16) int8_t Bs[kS8Tile][kS8K + 16];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int wm = (warp >> 2) * 64, wn = (warp & 3) * 32;
    int acc[4][4][4];
#pragma unroll
    for (int mi = 0; mi < 4; ++mi)
#pragma unroll
        for (int ni = 0; ni < 4; ++ni)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[mi][ni][e] = 0;
    for (int k0 = 0; k0 < K; k0 += kS8K) {
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            const int idx = tid + q * 256, row = idx >> 2, c16 = (idx & 3) * 16;
            *reinterpret_cast<int4 *>(&As[row][c16]) = __ldcg(reinterpret_cast<const int4 *>(Ag + row * ld + k0 + c16));
            *reinterpret_cast<int4 *>(&Bs[row][c16]) = __ldcg(reinterpret_cast<const int4 *>(Bg + row * ld + k0 + c16));
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < kS8K; kk += 32) {
            int a[4][4], b[4][2];
#pragma unroll
            for (int mi = 0; mi < 4; ++mi) {
                const int r = wm + mi * 16 + g;
                a[mi][0] = *reinterpret_cast<const int *>(&As[r][kk + t * 4]);
                a[mi][1] = *reinterpret_cast<const int *>(&As[r + 8][kk + t * 4]);
                a[mi][2] = *reinterpret_cast<const int *>(&As[r][kk + 16 + t * 4]);
                a[mi][3] = *reinterpret_cast<const int *>(&As[r + 8][kk + 16 + t * 4]);
            }
#pragma unroll
            for (int ni = 0; ni < 4; ++ni) {
                const int c = wn + ni * 8 + g;
                b[ni][0] = *reinterpret_cast<const int *>(&Bs[c][kk + t * 4]);
                b[ni][1] = *reinterpret_cast<const int *>(&Bs[c][kk + 16 + t * 4]);
            }
#pragma unroll
            for (int mi = 0; mi < 4; ++mi)
#pragma unroll
                for (int ni = 0; ni < 4; ++ni) imma_m16n8k32(acc[mi][ni], a[mi], b[ni]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int mi = 0; mi < 4; ++mi)
#pragma unroll
        for (int ni = 0; ni < 4; ++ni)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int r = wm + mi * 16 + g + (e >> 1) * 8;
                const int c = wn + ni * 8 + t * 2 + (e & 1);
                if (r >= nr || c >= nc) continue;
                if (!kAdd) Gt[(long long)r * ldg + c] = (double)acc[mi][ni][e] * unit;
                else if (acc[mi][ni][e] != 0) Gt[(long long)r * ldg + c] += (double)acc[mi][ni][e] * unit;
            }
}

// G[tile bi, tile bj] += unit * (image rows of bi) . (image rows of bj)^T over the chunk's K columns (lower triangle, bi >= bj)
__global__ void __launch_bounds__(256) ease_gram_s8_kernel(const int8_t *__restrict__ img, long long ld, int K, double *__restrict__ G,
                                                           int n, double unit)
{
    int bi, bj;
    tri_pair(blockIdx.x, bi, bj);
    gram_s8_tile<true>(img + (long long)bi * kS8Tile * ld, img + (long long)bj * kS8Tile * ld, ld, K,
                 G + (long long)bi * kS8Tile * n + (long long)bj * kS8Tile, n, n - bi * kS8Tile, n - bj * kS8Tile, unit);
}

// general path: Gt[r][c] += (64 fp64 image rows at Ag) . (64 rows at Bg)^T on DMMA for r < nr, c < nc (as gram_s8_tile;
// = when !kAdd)
template <bool kAdd>
__device__ __forceinline__ void gram_f64_tile(const double *__restrict__ Ag, const double *__restrict__ Bg, long long ld, int K,
                                              double *__restrict__ Gt, long long ldg, int nr, int nc)
{
    __shared__ DmmaSmem sm;
    double acc[4][2][2] = {};
    dmma_nt_64(Ag, ld, Bg, ld, K, acc, sm);
#pragma unroll
    for (int mi = 0; mi < 4; ++mi)
#pragma unroll
        for (int ni = 0; ni < 2; ++ni)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int r = dmma_row(mi), c = dmma_col(ni, e);
                if (r < nr && c < nc) {
                    if (kAdd) Gt[(long long)r * ldg + c] += acc[mi][ni][e];
                    else Gt[(long long)r * ldg + c] = acc[mi][ni][e];
                }
            }
}

// G[tile bi, tile bj] += (fp64 image rows of bi) . (rows of bj)^T (lower triangle)
__global__ void __launch_bounds__(256) ease_gram_f64_kernel(const double *__restrict__ img, long long ld, int K, double *__restrict__ G,
                                                            int n)
{
    int bi, bj;
    tri_pair(blockIdx.x, bi, bj);
    gram_f64_tile<true>(img + (long long)bi * kDmmaTile * ld, img + (long long)bj * kDmmaTile * ld, ld, K,
                  G + (long long)bi * kDmmaTile * n + (long long)bj * kDmmaTile, n, n - bi * kDmmaTile, n - bj * kDmmaTile);
}

// rectangular grid (column tiles, row tiles): G[r][c] = image row (p0 + r) . image row c for r < rows, c < n (G: ldg = n)
__global__ void __launch_bounds__(256) gram_panel_s8_kernel(const int8_t *__restrict__ img, long long ld, int K, int p0, int rows,
                                                            int n, double *__restrict__ G, double unit)
{
    const int r0 = blockIdx.y * kS8Tile, c0 = blockIdx.x * kS8Tile;
    gram_s8_tile<false>(img + (long long)(p0 + r0) * ld, img + (long long)c0 * ld, ld, K, G + (long long)r0 * n + c0, n, rows - r0, n - c0,
                 unit);
}

__global__ void __launch_bounds__(256) gram_panel_f64_kernel(const double *__restrict__ img, long long ld, int K, int p0, int rows,
                                                             int n, double *__restrict__ G)
{
    const int r0 = blockIdx.y * kDmmaTile, c0 = blockIdx.x * kDmmaTile;
    gram_f64_tile<false>(img + (long long)(p0 + r0) * ld, img + (long long)c0 * ld, ld, K, G + (long long)r0 * n + c0, n, rows - r0, n - c0);
}

// upper triangle := lower triangle; diagonal += reg (fp64, rounded once as scipy's G + reg * identity)
__global__ void ease_mirror_kernel(double *__restrict__ G, int n, double reg)
{
    const long long total = (long long)n * n;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < total; k += (long long)gridDim.x * blockDim.x) {
        const int i = (int)(k / n), j = (int)(k % n);
        if (i > j) G[(long long)j * n + i] = G[k];
        else if (i == j) G[k] += reg;
    }
}

// ---------------------------------------------------------------- sweep
// One CTA: the m x m diagonal block k0 (read from the lower triangle) swept in shared memory -> -D = -G_kk^-1, written
// over the block (full) and, negated, into D (kNb x kNb, zero outside m x m).  flag <- 1 on a pivot that is not > 0.
constexpr int kSweepThreads = 1024;
constexpr int kLdM = kNb + 1;

__global__ void __launch_bounds__(kSweepThreads) ease_diag_sweep_kernel(double *__restrict__ G, int n, int k0, int m,
                                                                        double *__restrict__ D, int *__restrict__ flag)
{
    extern __shared__ double M[];      // [kNb][kLdM]
    __shared__ double cp[kNb], rp[kNb];
    const int tid = threadIdx.x;
    for (int idx = tid; idx < m * m; idx += kSweepThreads) {
        const int r = idx / m, c = idx % m;
        M[r * kLdM + c] = r >= c ? G[(long long)(k0 + r) * n + k0 + c] : G[(long long)(k0 + c) * n + k0 + r];
    }
    __syncthreads();
    for (int p = 0; p < m; ++p) {
        const double piv = M[p * kLdM + p];
        if (tid < m) {
            cp[tid] = M[tid * kLdM + p];
            rp[tid] = M[p * kLdM + tid];
        }
        if (tid == 0 && !(piv > 0.0)) *flag = 1;
        __syncthreads();
        const double d = 1.0 / piv;
        for (int idx = tid; idx < m * m; idx += kSweepThreads) {
            const int i = idx / m, j = idx % m;
            double v;
            if (i != p && j != p) v = M[i * kLdM + j] - cp[i] * rp[j] * d;
            else if (i == p && j == p) v = -d;
            else if (i == p) v = rp[j] * d;
            else v = cp[i] * d;
            M[i * kLdM + j] = v;
        }
        __syncthreads();
    }
    for (int idx = tid; idx < kNb * kNb; idx += kSweepThreads) {
        const int r = idx / kNb, c = idx % kNb;
        const bool in = r < m && c < m;
        D[idx] = in ? -M[r * kLdM + c] : 0.0;
        if (in) G[(long long)(k0 + r) * n + k0 + c] = M[r * kLdM + c];
    }
}

// V[i][c] = G[i][k0 + c] for i outside the pivot block (read from the lower triangle), 0 elsewhere; V is n128 x kNb
__global__ void ease_gather_panel_kernel(const double *__restrict__ G, int n, int k0, int m, long long n128, double *__restrict__ V)
{
    const long long total = n128 * kNb;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < total; k += (long long)gridDim.x * blockDim.x) {
        const int i = (int)(k / kNb), c = (int)(k % kNb);
        double v = 0.0;
        if (i < n && c < m && (i < k0 || i >= k0 + m)) {
            const int j = k0 + c;
            v = i > j ? G[(long long)i * n + j] : G[(long long)j * n + i];
        }
        V[k] = v;
    }
}

// W = V D (D symmetric: W_ic = sum_m V_im D_cm); also the swept panel: G[i][k0 + c] (i below the block) or G[k0 + c][i]
// (i above it) = W_ic.  Grid: (n128 / 64, kNb / 64).
__global__ void __launch_bounds__(256) ease_panel_kernel(const double *__restrict__ V, const double *__restrict__ D,
                                                         double *__restrict__ W, double *__restrict__ G, int n, int k0, int m)
{
    __shared__ DmmaSmem sm;
    const int rt = blockIdx.x, ct = blockIdx.y;
    double acc[4][2][2] = {};
    dmma_nt_64(V + (long long)rt * kDmmaTile * kNb, kNb, D + (long long)ct * kDmmaTile * kNb, kNb, kNb, acc, sm);
#pragma unroll
    for (int mi = 0; mi < 4; ++mi)
#pragma unroll
        for (int ni = 0; ni < 2; ++ni)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int i = rt * kDmmaTile + dmma_row(mi), c = ct * kDmmaTile + dmma_col(ni, e);
                const double v = acc[mi][ni][e];
                W[(long long)i * kNb + c] = v;
                if (i < n && c < m && (i < k0 || i >= k0 + m)) {
                    const int j = k0 + c;
                    if (i > j) G[(long long)i * n + j] = v; else G[(long long)j * n + i] = v;
                }
            }
}

// rank-kNb update of the lower tiles outside the pivot block: G_IJ -= W_I V_J^T (64 x 64 tiles, I >= J)
__global__ void __launch_bounds__(256) ease_update_kernel(const double *__restrict__ W, const double *__restrict__ V,
                                                          double *__restrict__ G, int n, int kt0, int kt1)
{
    __shared__ DmmaSmem sm;
    int bi, bj;
    tri_pair(blockIdx.x, bi, bj);
    if ((bi >= kt0 && bi < kt1) || (bj >= kt0 && bj < kt1)) return;   // uniform across the CTA
    double acc[4][2][2] = {};
    dmma_nt_64(W + (long long)bi * kDmmaTile * kNb, kNb, V + (long long)bj * kDmmaTile * kNb, kNb, kNb, acc, sm);
#pragma unroll
    for (int mi = 0; mi < 4; ++mi)
#pragma unroll
        for (int ni = 0; ni < 2; ++ni)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int r = bi * kDmmaTile + dmma_row(mi), c = bj * kDmmaTile + dmma_col(ni, e);
                if (r < n && c < n) G[(long long)r * n + c] -= acc[mi][ni][e];
            }
}

// the swept matrix holds -P in its lower triangle: P = negated lower, mirrored
__global__ void ease_negate_mirror_kernel(double *__restrict__ G, int n)
{
    const long long total = (long long)n * n;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < total; k += (long long)gridDim.x * blockDim.x) {
        const int i = (int)(k / n), j = (int)(k % n);
        if (i < j) continue;
        const double v = -G[k];
        G[k] = v;
        if (i > j) G[(long long)j * n + i] = v;
    }
}

__global__ void ease_diag_kernel(const double *__restrict__ P, int n, double *__restrict__ diag)
{
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) diag[i] = P[(long long)i * n + i];
}

// B = -P / diag(P) (numpy divides column j by P_jj), zero diagonal
__global__ void ease_weights_kernel(double *__restrict__ P, int n, const double *__restrict__ diag)
{
    const long long total = (long long)n * n;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < total; k += (long long)gridDim.x * blockDim.x) {
        const int i = (int)(k / n), j = (int)(k % n);
        P[k] = i == j ? 0.0 : -P[k] / diag[j];
    }
}

// ---------------------------------------------------------------- scoring
constexpr int kRankThreads = 256;

// one CTA per test user: s_c = sum_{i in row(u)} x_ui B[cand_c, i] (warp per candidate), then top-k of the C scores
__global__ void __launch_bounds__(kRankThreads) ease_rank_kernel(const double *__restrict__ B, int n, const int64_t *__restrict__ row_ptr,
                                                                 const int32_t *__restrict__ col, const float *__restrict__ val,
                                                                 const int64_t *__restrict__ users, const int64_t *__restrict__ cands,
                                                                 int C, int k, int64_t *__restrict__ out, double *__restrict__ scores)
{
    extern __shared__ double sc[];
    const int row = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long u = users[row], b = row_ptr[u], e = row_ptr[u + 1];
    const int64_t *cr = cands + (long long)row * C;
    for (int c = warp; c < C; c += kRankThreads / 32) {
        const double *Brow = B + cr[c] * n;
        double acc = 0.0;
        for (long long q = b + lane; q < e; q += 32) acc += (double)val[q] * Brow[col[q]];
        acc = warp_sum(acc);
        if (lane == 0) {
            sc[c] = acc;
            if (scores) scores[(long long)row * C + c] = acc;
        }
    }
    __syncthreads();
    block_topk(sc, C, k, cr, out + (long long)row * k);
}

// scores[row][j] = sum_{i in row(u)} x_ui B[i, j]: thread per item j, the user's items in ascending order (coalesced rows of B)
__global__ void ease_user_scores_kernel(const double *__restrict__ B, int n, const int64_t *__restrict__ row_ptr,
                                        const int32_t *__restrict__ col, const float *__restrict__ val,
                                        const int64_t *__restrict__ users, double *__restrict__ scores)
{
    const int j = blockIdx.x * blockDim.x + threadIdx.x, row = blockIdx.y;
    if (j >= n) return;
    const long long u = users[row];
    double acc = 0.0;
    for (long long q = row_ptr[u]; q < row_ptr[u + 1]; ++q) acc += (double)val[q] * B[(long long)col[q] * n + j];
    scores[(long long)row * n + j] = acc;
}

__global__ void __launch_bounds__(1024) ease_full_topk_kernel(const double *__restrict__ scores, int n, int k, int64_t *__restrict__ out)
{
    block_topk(scores + (long long)blockIdx.x * n, n, k, nullptr, out + (long long)blockIdx.x * k);
}

// out[p] = sum_{i in row(u_p)} x_ui B[i, j_p]; warp per pair
__global__ void ease_predict_kernel(const double *__restrict__ B, int n, const int64_t *__restrict__ row_ptr,
                                    const int32_t *__restrict__ col, const float *__restrict__ val, const int64_t *__restrict__ users,
                                    const int64_t *__restrict__ items, long long n_pairs, double *__restrict__ out)
{
    const int lane = threadIdx.x & 31;
    for (long long p = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; p < n_pairs;
         p += ((long long)gridDim.x * blockDim.x) >> 5) {
        const long long u = users[p], j = items[p];
        double acc = 0.0;
        for (long long q = row_ptr[u] + lane; q < row_ptr[u + 1]; q += 32) acc += (double)val[q] * B[(long long)col[q] * n + j];
        acc = warp_sum(acc);
        if (lane == 0) out[p] = acc;
    }
}

// the exact-Gram rule on the gathered statistics (drb_ease_csr's comment above); synchronises
static int exact_scale(const double *colsq, int item_num, CsrStats *stats, int32_t *h_scale, cudaStream_t st)
{
    ease_sqmax_kernel<<<grid_for(item_num, 256), 256, 0, st>>>(colsq, item_num, stats);
    DRB_CUDA(cudaGetLastError());
    CsrStats h;
    DRB_CUDA(cudaMemcpyAsync(&h, stats, sizeof(h), cudaMemcpyDeviceToHost, st));
    DRB_CUDA(cudaStreamSynchronize(st));
    int s = -1;
    if (h.smax <= 7) {
        uint32_t a = h.amax;
        float amax;
        memcpy(&amax, &a, sizeof(amax));
        double sq;
        memcpy(&sq, &h.sqmax, sizeof(sq));
        if ((double)amax * (double)(1 << h.smax) <= 127.0 && sq * (double)(1 << (2 * h.smax)) < 2147483648.0) s = (int)h.smax;
    }
    *h_scale = s;
    return DRB_OK;
}

}  // namespace drb

using namespace drb;

extern "C" size_t drb_ease_csr_workspace_bytes(int32_t item_num, int64_t nnz)
{
    if (item_num <= 0 || nnz < 0) return 0;
    return 256 + round_up(sizeof(double) * (size_t)item_num, 256) + sizeof(double) * (size_t)(nnz > 0 ? nnz : 1);
}

extern "C" int drb_ease_csr(const int64_t *d_seq_ptr, const int32_t *d_order, const int32_t *d_coo_i, const double *d_coo_v,
                            int32_t user_num, int32_t item_num, const int64_t *d_row_ptr, const int32_t *d_col, int64_t nnz,
                            void *d_ws, float *d_val, int32_t *h_scale, void *stream)
{
    DRB_REQUIRE(d_seq_ptr && d_row_ptr && d_ws && h_scale && user_num > 0 && item_num > 0 && nnz >= 0 &&
                    (nnz == 0 || (d_order && d_coo_i && d_coo_v && d_col && d_val)),
                "ease_csr: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    CsrStats *stats = (CsrStats *)d_ws;
    double *colsq = (double *)((char *)d_ws + 256);
    double *sum = (double *)((char *)d_ws + 256 + round_up(sizeof(double) * (size_t)item_num, 256));
    DRB_CUDA(cudaMemsetAsync(d_ws, 0, 256 + sizeof(double) * (size_t)item_num, st));
    ease_values_kernel<<<grid_for(user_num, 128), 128, 0, st>>>(d_seq_ptr, d_order, d_coo_i, d_coo_v, user_num, d_row_ptr, d_col,
                                                                 sum, d_val, colsq, stats);
    return exact_scale(colsq, item_num, stats, h_scale, st);
}

extern "C" int drb_ease_scale(const int64_t *d_row_ptr, const int32_t *d_col, const float *d_val, int32_t user_num,
                              int32_t item_num, void *d_ws, int32_t *h_scale, void *stream)
{
    DRB_REQUIRE(d_row_ptr && d_ws && h_scale && user_num > 0 && item_num > 0, "ease_scale: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    CsrStats *stats = (CsrStats *)d_ws;
    double *colsq = (double *)((char *)d_ws + 256);
    DRB_CUDA(cudaMemsetAsync(d_ws, 0, 256 + sizeof(double) * (size_t)item_num, st));
    ease_stats_kernel<<<grid_for(user_num, 128), 128, 0, st>>>(d_row_ptr, d_col, d_val, user_num, colsq, stats);
    return exact_scale(colsq, item_num, stats, h_scale, st);
}

extern "C" size_t drb_ease_workspace_bytes(int32_t user_num, int32_t item_num, int32_t scale)
{
    if (user_num <= 0 || item_num <= 0) return 0;
    return carve_ease(nullptr, user_num, item_num, scale, nullptr);
}

extern "C" int drb_ease_gram(const int64_t *d_row_ptr, const int32_t *d_col, const float *d_val, int32_t user_num, int32_t item_num,
                             int32_t scale, double reg, void *d_ws, double *d_G, void *stream)
{
    DRB_REQUIRE(d_row_ptr && d_ws && d_G && user_num > 0 && item_num > 0 && scale <= 7, "ease_gram: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    EaseWs w;
    carve_ease(d_ws, user_num, item_num, scale, &w);
    const EaseGeom g = ease_geom(user_num, item_num, scale);
    const int n = item_num;
    DRB_CUDA(cudaMemsetAsync(d_G, 0, sizeof(double) * (size_t)n * n, st));
    const bool exact = scale >= 0;
    const size_t img_bytes = (size_t)(g.rows * g.chunk * (exact ? 1 : 8));
    const long long tiles = g.rows / (exact ? kS8Tile : kDmmaTile), pairs = tiles * (tiles + 1) / 2;
    DRB_REQUIRE(pairs < (1ll << 31), "ease_gram: %d items exceed the tile grid", n);
    for (long long u0 = 0; u0 < user_num; u0 += g.chunk) {
        const int u1 = (int)(u0 + g.chunk < user_num ? u0 + g.chunk : user_num);
        DRB_CUDA(cudaMemsetAsync(w.image, 0, img_bytes, st));
        const int grid = grid_for((long long)(u1 - u0) * 32, 256);
        if (exact) {
            ease_image_kernel<int8_t><<<grid, 256, 0, st>>>(d_row_ptr, d_col, d_val, (int)u0, u1, g.chunk, (float)(1 << scale),
                                                             (int8_t *)w.image);
            ease_gram_s8_kernel<<<(unsigned)pairs, 256, 0, st>>>((const int8_t *)w.image, g.chunk, (int)g.chunk, d_G, n,
                                                                 ldexp(1.0, -2 * scale));
        } else {
            ease_image_kernel<double><<<grid, 256, 0, st>>>(d_row_ptr, d_col, d_val, (int)u0, u1, g.chunk, 1.f, (double *)w.image);
            ease_gram_f64_kernel<<<(unsigned)pairs, 256, 0, st>>>((const double *)w.image, g.chunk, (int)g.chunk, d_G, n);
        }
        DRB_CUDA(cudaGetLastError());
    }
    ease_mirror_kernel<<<grid_for((long long)n * n, 256), 256, 0, st>>>(d_G, n, reg);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}

// the whole-K image of drb_gram_image: rows = the CSR's columns padded to the s8 tile, ld = its rows padded to the K step
static void panel_geom(int K, int n, long long &rows, long long &ld)
{
    rows = round_up(n, kS8Tile);
    ld = round_up(K, kS8K);
}

extern "C" size_t drb_gram_image_bytes(int32_t k_rows, int32_t n, int32_t scale)
{
    if (k_rows <= 0 || n <= 0) return 0;
    long long rows, ld;
    panel_geom(k_rows, n, rows, ld);
    return (size_t)(rows * ld * (scale >= 0 ? 1 : 8));
}

extern "C" int drb_gram_image(const int64_t *d_row_ptr, const int32_t *d_col, const float *d_val, int32_t k_rows, int32_t n,
                              int32_t scale, void *d_img, void *stream)
{
    DRB_REQUIRE(d_row_ptr && d_img && k_rows > 0 && n > 0 && scale <= 7, "gram_image: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    long long rows, ld;
    panel_geom(k_rows, n, rows, ld);
    DRB_CUDA(cudaMemsetAsync(d_img, 0, drb_gram_image_bytes(k_rows, n, scale), st));
    const int grid = grid_for((long long)k_rows * 32, 256);
    if (scale >= 0)
        ease_image_kernel<int8_t><<<grid, 256, 0, st>>>(d_row_ptr, d_col, d_val, 0, k_rows, ld, (float)(1 << scale), (int8_t *)d_img);
    else
        ease_image_kernel<double><<<grid, 256, 0, st>>>(d_row_ptr, d_col, d_val, 0, k_rows, ld, 1.f, (double *)d_img);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}

extern "C" int drb_gram_panel(const void *d_img, int32_t k_rows, int32_t n, int32_t scale, int32_t p0, int32_t rows, double *d_G,
                              void *stream)
{
    DRB_REQUIRE(d_img && d_G && k_rows > 0 && n > 0 && scale <= 7 && p0 >= 0 && p0 % kS8Tile == 0 && rows > 0 && p0 + rows <= n,
                "gram_panel: bad arguments (p0 a multiple of %d, p0 + rows <= n)", kS8Tile);
    cudaStream_t st = (cudaStream_t)stream;
    long long prow, ld;
    panel_geom(k_rows, n, prow, ld);
    const int T = scale >= 0 ? kS8Tile : kDmmaTile;
    const dim3 grid((unsigned)((n + T - 1) / T), (unsigned)((rows + T - 1) / T));
    DRB_REQUIRE(grid.y <= 65535, "gram_panel: %d rows exceed the tile grid", rows);
    if (scale >= 0)
        gram_panel_s8_kernel<<<grid, 256, 0, st>>>((const int8_t *)d_img, ld, (int)ld, p0, rows, n, d_G, ldexp(1.0, -2 * scale));
    else
        gram_panel_f64_kernel<<<grid, 256, 0, st>>>((const double *)d_img, ld, (int)ld, p0, rows, n, d_G);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}

extern "C" int drb_ease_inverse(double *d_G, int32_t item_num, void *d_ws, void *stream)
{
    DRB_REQUIRE(d_G && d_ws && item_num > 0, "ease_inverse: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    EaseWs w;
    carve_ease(d_ws, 1, item_num, 0, &w);
    const EaseGeom g = ease_geom(1, item_num, 0);
    const int n = item_num;
    const long long tiles = (n + kDmmaTile - 1) / kDmmaTile, pairs = tiles * (tiles + 1) / 2;
    DRB_REQUIRE(pairs < (1ll << 31), "ease_inverse: %d items exceed the tile grid", n);
    const size_t smem = sizeof(double) * kNb * kLdM;
    DRB_CUDA(cudaFuncSetAttribute(ease_diag_sweep_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    DRB_CUDA(cudaMemsetAsync(w.flag, 0, sizeof(int), st));
    for (int k0 = 0; k0 < n; k0 += kNb) {
        const int m = n - k0 < kNb ? n - k0 : kNb;
        ease_diag_sweep_kernel<<<1, kSweepThreads, smem, st>>>(d_G, n, k0, m, w.D, w.flag);
        ease_gather_panel_kernel<<<grid_for(g.n128 * kNb, 256), 256, 0, st>>>(d_G, n, k0, m, g.n128, w.V);
        ease_panel_kernel<<<dim3((unsigned)(g.n128 / kDmmaTile), kNb / kDmmaTile), 256, 0, st>>>(w.V, w.D, w.W, d_G, n, k0, m);
        ease_update_kernel<<<(unsigned)pairs, 256, 0, st>>>(w.W, w.V, d_G, n, k0 / kDmmaTile, (k0 + m + kDmmaTile - 1) / kDmmaTile);
        DRB_CUDA(cudaGetLastError());
    }
    ease_negate_mirror_kernel<<<grid_for((long long)n * n, 256), 256, 0, st>>>(d_G, n);
    DRB_CUDA(cudaGetLastError());
    int flag = 0;
    DRB_CUDA(cudaMemcpyAsync(&flag, w.flag, sizeof(int), cudaMemcpyDeviceToHost, st));
    DRB_CUDA(cudaStreamSynchronize(st));
    if (flag) {
        set_error("ease_inverse: G + reg I is not positive definite (a pivot <= 0)");
        return DRB_ERR_NOT_PD;
    }
    return DRB_OK;
}

extern "C" int drb_ease_weights(double *d_P, int32_t item_num, void *d_ws, void *stream)
{
    DRB_REQUIRE(d_P && d_ws && item_num > 0, "ease_weights: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    EaseWs w;
    carve_ease(d_ws, 1, item_num, 0, &w);
    const int n = item_num;
    ease_diag_kernel<<<grid_for(n, 256), 256, 0, st>>>(d_P, n, w.diag);
    ease_weights_kernel<<<grid_for((long long)n * n, 256), 256, 0, st>>>(d_P, n, w.diag);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}

extern "C" int drb_ease_rank(const double *d_B, int32_t item_num, const int64_t *d_row_ptr, const int32_t *d_col, const float *d_val,
                             const int64_t *d_users, int64_t n_users, const int64_t *d_cands, int32_t cand_num, int32_t topk,
                             int64_t *d_out, double *d_scores, void *stream)
{
    DRB_REQUIRE(d_B && d_row_ptr && d_users && d_cands && d_out && item_num > 0 && n_users >= 0 && cand_num > 0 && topk > 0 &&
                    topk <= cand_num,
                "ease_rank: bad arguments");
    const size_t smem = sizeof(double) * (size_t)cand_num;
    DRB_REQUIRE(smem <= 200 * 1024, "ease_rank: %d candidates exceed shared memory", cand_num);
    if (n_users == 0) return DRB_OK;
    if (smem > 48 * 1024) DRB_CUDA(cudaFuncSetAttribute(ease_rank_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    DRB_REQUIRE(n_users < (1ll << 31), "ease_rank: too many users");
    ease_rank_kernel<<<(unsigned)n_users, kRankThreads, smem, (cudaStream_t)stream>>>(d_B, item_num, d_row_ptr, d_col, d_val, d_users,
                                                                                     d_cands, cand_num, topk, d_out, d_scores);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}

extern "C" int drb_ease_full_rank(const double *d_B, int32_t item_num, const int64_t *d_row_ptr, const int32_t *d_col,
                                  const float *d_val, const int64_t *d_users, int32_t n_users, int32_t topk, double *d_scores,
                                  int64_t *d_out, void *stream)
{
    DRB_REQUIRE(d_B && d_row_ptr && d_users && d_scores && d_out && item_num > 0 && n_users >= 0 && topk > 0 && topk <= item_num &&
                    n_users <= 65535,
                "ease_full_rank: bad arguments");
    if (n_users == 0) return DRB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    ease_user_scores_kernel<<<dim3((item_num + 255) / 256, n_users), 256, 0, st>>>(d_B, item_num, d_row_ptr, d_col, d_val, d_users,
                                                                                   d_scores);
    ease_full_topk_kernel<<<n_users, 1024, 0, st>>>(d_scores, item_num, topk, d_out);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}

extern "C" int drb_ease_predict(const double *d_B, int32_t item_num, const int64_t *d_row_ptr, const int32_t *d_col,
                                const float *d_val, const int64_t *d_users, const int64_t *d_items, int64_t n_pairs, double *d_out,
                                void *stream)
{
    DRB_REQUIRE(d_B && d_row_ptr && d_users && d_items && d_out && item_num > 0 && n_pairs >= 0, "ease_predict: bad arguments");
    if (n_pairs == 0) return DRB_OK;
    ease_predict_kernel<<<grid_for(n_pairs * 32, 256), 256, 0, (cudaStream_t)stream>>>(d_B, item_num, d_row_ptr, d_col, d_val, d_users,
                                                                                      d_items, n_pairs, d_out);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}
