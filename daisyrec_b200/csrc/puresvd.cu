// puresvd.cu -- PureSVD (daisy/model/PureSVDRecommender.py) on the device.
//
// The reference's fit is sklearn's randomized_svd(X, factors, random_state=2019) on the host: l = factors + 10 random
// directions Omega, n_iter power rounds Q = LU(A Q), Q = LU(A^T Q), Q = qr(A Q), B = Q^T A, svd(B), svd_flip; A = X^T when
// U < I.  Here every normaliser is shifted CholeskyQR3 (the same subspace as LU or QR), and the projected SVD is taken as
// B^T = A^T Q = Q_b R, R^T = Ur S Vr^T (one-sided Jacobi), U_A = Q Ur, V_A = Q_b Vr.  All arithmetic is fp64 and every sum
// runs in a fixed order without floating-point atomics, so two fits are bitwise equal.
//
//   drb_puresvd_csr        X's fp64 values (duplicates summed in row order, as scipy's csr_matrix up to the order of three or
//                          more duplicates) and the values of the item-major CSR of X^T, so that both A Z and A^T Z are gathers.
//   drb_puresvd_spmm       Y[r, :] = sum_j A[r, j] Z[j, :] over one CSR for a row-major fp64 panel; each output row summed in
//                          CSR order by one warp (lanes over columns), rows longer than kLongRow by a CTA whose warps sum
//                          contiguous segments, added in warp order.
//   drb_puresvd_orth       shifted CholeskyQR3 of a panel Y [m, l] in place: three passes of W = Y^T Y (+ s I on the first,
//                          s = 11 (m l + l (l + 1)) u ||Y||_F^2), Cholesky W = R^T R in one CTA, Y <- Y R^-1.  Gram and
//                          Y R^-1 on DMMA; the Gram's row chunks give l x l partials summed in chunk order.  The padded
//                          columns get an identity Gram.  DRB_ERR_NOT_PD on a pivot <= l u max_j W_jj.
//   drb_puresvd_small_svd  one-sided Jacobi SVD of R^T (l x l) in one CTA on global (L2-resident) buffers: disjoint column
//                          pairs rotated in a fixed round-robin order, sweeps until every pair is orthogonal to fp64 precision
//                          (no pair of a sweep with |cos| above l eps).
//   drb_puresvd_factors    U_A = Q Ur, V_A = Q_b Vr on DMMA for the k largest sigma, the user-side sign rule, item side x sigma.
//   drb_puresvd_scores     user_vec[u] . item_vec[c] (lanes over k, a fixed butterfly), for candidates or every item.
#include <math.h>

#include "common.cuh"
#include "dmma.cuh"

namespace drb {

constexpr double kUnit = 0x1p-53;      // fp64 unit roundoff
constexpr int kLongRow = 2048;         // rows longer than this are summed by a CTA
constexpr int kLongWarps = 16;
constexpr int kSpmmCols = 8;           // column chunks of 32 per lane and pass
constexpr int kCholThreads = 1024;
constexpr int kJacobiThreads = 1024;
constexpr int kMaxSweeps = 60;

static long long round_up(long long x, long long m) { return (x + m - 1) / m * m; }

// ---------------------------------------------------------------- X and X^T
// one thread per user: each CSR slot's COO values summed in fp64 in row order (d_order: rows grouped by user, stable)
__global__ void psvd_values_kernel(const int64_t *__restrict__ seq_ptr, const int32_t *__restrict__ order,
                                   const int32_t *__restrict__ coo_i, const double *__restrict__ coo_v, int U,
                                   const int64_t *__restrict__ row_ptr, const int32_t *__restrict__ col, double *__restrict__ val)
{
    for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < U; u += gridDim.x * blockDim.x) {
        const long long b = row_ptr[u], e = row_ptr[u + 1];
        for (long long k = b; k < e; ++k) val[k] = 0.0;
        for (long long q = seq_ptr[u]; q < seq_ptr[u + 1]; ++q) {
            const int r = order[q];
            const int item = coo_i[r];
            long long lo = b, hi = e - 1;
            while (lo < hi) {
                const long long mid = (lo + hi) >> 1;
                if (col[mid] < item) lo = mid + 1; else hi = mid;
            }
            val[lo] += coo_v[r];
        }
    }
}

// slot k of X^T (item it, user t_col[k]): the value of slot (user, it) of X, found by binary search in both CSRs
__global__ void psvd_transpose_kernel(const int64_t *__restrict__ row_ptr, const int32_t *__restrict__ col,
                                      const double *__restrict__ val, const int64_t *__restrict__ t_ptr,
                                      const int32_t *__restrict__ t_col, int I, long long nnz, double *__restrict__ t_val)
{
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < nnz; k += (long long)gridDim.x * blockDim.x) {
        int lo = 0, hi = I;                 // the item: the last it with t_ptr[it] <= k
        while (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if (t_ptr[mid] <= k) lo = mid; else hi = mid;
        }
        const int item = lo, u = t_col[k];
        long long a = row_ptr[u], b = row_ptr[u + 1] - 1;   // the pair is in the row: both CSRs hold the same pairs
        while (a < b) {
            const long long mid = (a + b) >> 1;
            if (col[mid] < item) a = mid + 1; else b = mid;
        }
        t_val[k] = val[a];
    }
}

// ---------------------------------------------------------------- SpMM
// acc[j] += sum over the CSR slots [b, e) of a_k Z[col_k, c0 + lane + 32 j], in slot order
template <int NC>
__device__ __forceinline__ void spmm_segment(const int32_t *__restrict__ col, const double *__restrict__ val, long long b,
                                             long long e, const double *__restrict__ Z, long long ld, int c0, int l,
                                             double (&acc)[NC])
{
    const int lane = threadIdx.x & 31;
    long long k = b;
    for (; k + 4 <= e; k += 4) {
        double a[4], z[4][NC];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            a[q] = val[k + q];
            const double *zr = Z + (long long)col[k + q] * ld + c0 + lane;
#pragma unroll
            for (int j = 0; j < NC; ++j) z[q][j] = c0 + lane + 32 * j < l ? zr[32 * j] : 0.0;
        }
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
            for (int j = 0; j < NC; ++j) acc[j] = __fma_rn(a[q], z[q][j], acc[j]);
    }
    for (; k < e; ++k) {
        const double a = val[k];
        const double *zr = Z + (long long)col[k] * ld + c0 + lane;
#pragma unroll
        for (int j = 0; j < NC; ++j)
            if (c0 + lane + 32 * j < l) acc[j] = __fma_rn(a, zr[32 * j], acc[j]);
    }
}

// a warp per row of at most kLongRow slots; writes columns [c0, c0 + 32 NC) of the row (zero at and past l)
template <int NC>
__global__ void __launch_bounds__(256) psvd_spmm_kernel(const int64_t *__restrict__ row_ptr, const int32_t *__restrict__ col,
                                                        const double *__restrict__ val, int n_rows, const double *__restrict__ Z,
                                                        long long ld, int c0, int l, double *__restrict__ Y)
{
    const int lane = threadIdx.x & 31;
    for (long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n_rows;
         r += ((long long)gridDim.x * blockDim.x) >> 5) {
        const long long b = row_ptr[r], e = row_ptr[r + 1];
        if (e - b > kLongRow) continue;
        double acc[NC];
#pragma unroll
        for (int j = 0; j < NC; ++j) acc[j] = 0.0;
        spmm_segment<NC>(col, val, b, e, Z, ld, c0, l, acc);
#pragma unroll
        for (int j = 0; j < NC; ++j) {
            const int c = c0 + lane + 32 * j;
            if (c < ld) Y[r * ld + c] = c < l ? acc[j] : 0.0;
        }
    }
}

// a CTA per row longer than kLongRow: warp w sums the w-th contiguous segment, the segments are added in warp order
template <int NC>
__global__ void __launch_bounds__(kLongWarps * 32) psvd_spmm_long_kernel(const int64_t *__restrict__ row_ptr,
                                                                         const int32_t *__restrict__ col,
                                                                         const double *__restrict__ val, int n_rows,
                                                                         const double *__restrict__ Z, long long ld, int c0,
                                                                         int l, double *__restrict__ Y)
{
    __shared__ double part[kLongWarps][NC * 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (long long r = blockIdx.x; r < n_rows; r += gridDim.x) {
        const long long b = row_ptr[r], e = row_ptr[r + 1];
        if (e - b <= kLongRow) continue;                    // uniform across the CTA
        const long long seg = (e - b + kLongWarps - 1) / kLongWarps;
        const long long sb = b + warp * seg, se = sb + seg < e ? sb + seg : e;
        double acc[NC];
#pragma unroll
        for (int j = 0; j < NC; ++j) acc[j] = 0.0;
        if (sb < se) spmm_segment<NC>(col, val, sb, se, Z, ld, c0, l, acc);
#pragma unroll
        for (int j = 0; j < NC; ++j) part[warp][lane + 32 * j] = acc[j];
        __syncthreads();
        for (int t = threadIdx.x; t < NC * 32; t += blockDim.x) {
            const int c = c0 + t;
            if (c >= ld) continue;
            double s = 0.0;
            for (int w = 0; w < kLongWarps; ++w) s += part[w][t];
            Y[r * ld + c] = c < l ? s : 0.0;
        }
        __syncthreads();
    }
}

template <int NC>
static void spmm_launch(const int64_t *row_ptr, const int32_t *col, const double *val, int n_rows, const double *Z, int ld,
                        int c0, int l, double *Y, cudaStream_t st)
{
    psvd_spmm_kernel<NC><<<grid_for((long long)n_rows * 32, 256), 256, 0, st>>>(row_ptr, col, val, n_rows, Z, ld, c0, l, Y);
    psvd_spmm_long_kernel<NC><<<grid_for(n_rows, 1, 8), kLongWarps * 32, 0, st>>>(row_ptr, col, val, n_rows, Z, ld, c0, l, Y);
}

// ---------------------------------------------------------------- orth
// partial Gram of row chunk z: part[z][tile bi, tile bj] = Y[rows of z, cols of bi]^T Y[rows of z, cols of bj] on DMMA.
// The operands are staged K-major (rows of Y) and the fragments read transposed; 72-double rows keep the 8 x 4 fragment
// reads on distinct bank pairs.
__global__ void __launch_bounds__(256) psvd_gram_kernel(const double *__restrict__ Y, long long mp, int ld, long long chunk,
                                                        double *__restrict__ part)
{
    __shared__ double sa[kDmmaK][kDmmaTile + 8];
    __shared__ double sb[kDmmaK][kDmmaTile + 8];
    const int bi = blockIdx.x, bj = blockIdx.y, z = blockIdx.z;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int wm = (warp >> 2) * 32, wn = (warp & 3) * 16;
    const long long r0 = (long long)z * chunk, r1 = r0 + chunk < mp ? r0 + chunk : mp;
    double acc[4][2][2] = {};
    for (long long k0 = r0; k0 < r1; k0 += kDmmaK) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int idx = tid + q * 256, kk = idx >> 5, c2 = (idx & 31) * 2;
            const double *row = Y + (k0 + kk) * ld;
            *reinterpret_cast<double2 *>(&sa[kk][c2]) = __ldcg(reinterpret_cast<const double2 *>(row + bi * kDmmaTile + c2));
            *reinterpret_cast<double2 *>(&sb[kk][c2]) = __ldcg(reinterpret_cast<const double2 *>(row + bj * kDmmaTile + c2));
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < kDmmaK; kk += 4) {
            double a[4], b[2];
#pragma unroll
            for (int mi = 0; mi < 4; ++mi) a[mi] = sa[kk + t][wm + mi * 8 + g];
#pragma unroll
            for (int ni = 0; ni < 2; ++ni) b[ni] = sb[kk + t][wn + ni * 8 + g];
#pragma unroll
            for (int mi = 0; mi < 4; ++mi)
#pragma unroll
                for (int ni = 0; ni < 2; ++ni) dmma_m8n8k4(acc[mi][ni], a[mi], b[ni]);
        }
        __syncthreads();
    }
    double *P = part + (long long)z * ld * ld;
#pragma unroll
    for (int mi = 0; mi < 4; ++mi)
#pragma unroll
        for (int ni = 0; ni < 2; ++ni)
#pragma unroll
            for (int e = 0; e < 2; ++e)
                P[(long long)(bi * kDmmaTile + dmma_row(mi)) * ld + bj * kDmmaTile + dmma_col(ni, e)] = acc[mi][ni][e];
}

// W = sum of the chunk partials in chunk order
__global__ void psvd_gram_reduce_kernel(const double *__restrict__ part, int nchunks, long long n2, double *__restrict__ W)
{
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n2; i += (long long)gridDim.x * blockDim.x) {
        double s = 0.0;
        for (int z = 0; z < nchunks; ++z) s += part[(long long)z * n2 + i];
        W[i] = s;
    }
}

// One CTA: the padded block of W set to the identity (and the shift added when asked), W = R^T R (R upper, in place,
// right-looking), Li = (R^T)^-1 = (R^-1)^T by a row sweep, and Racc <- R Racc (Racc <- R when first).  flag <- 1 on a
// pivot <= tau (NaN included).
__global__ void __launch_bounds__(kCholThreads) psvd_chol_kernel(double *__restrict__ W, int l, int ld, long long m, int shifted,
                                                                 double *__restrict__ Li, double *__restrict__ Racc,
                                                                 int racc_first, double *__restrict__ scratch,
                                                                 int *__restrict__ flag)
{
    __shared__ double s_tr, s_max;
    const int tid = threadIdx.x;
    if (tid == 0) {
        double tr = 0.0, mx = 0.0;
        for (int j = 0; j < l; ++j) {
            const double d = W[(long long)j * ld + j];
            tr += d;
            mx = fmax(mx, d);
        }
        s_tr = tr;
        s_max = mx;
    }
    __syncthreads();
    const double shift = shifted ? 11.0 * ((double)m * l + (double)l * (l + 1)) * kUnit * s_tr : 0.0;
    const double tau = l * kUnit * s_max;
    const long long n2 = (long long)ld * ld;
    for (long long idx = tid; idx < n2; idx += kCholThreads) {
        const int i = (int)(idx / ld), j = (int)(idx % ld);
        if (i >= l || j >= l) W[idx] = i == j ? 1.0 : 0.0;
        else if (i == j) W[idx] += shift;
    }
    __syncthreads();
    for (int p = 0; p < ld; ++p) {
        const double piv = W[(long long)p * ld + p];
        if (tid == 0 && p < l && !(piv > tau)) *flag = 1;
        const double r = sqrt(fmax(piv, 0.0)), rinv = 1.0 / r;
        __syncthreads();
        for (int j = p + tid; j < ld; j += kCholThreads) W[(long long)p * ld + j] = j == p ? r : W[(long long)p * ld + j] * rinv;
        __syncthreads();
        const int cnt = ld - p - 1;
        for (long long idx = tid; idx < (long long)cnt * cnt; idx += kCholThreads) {
            const int i = p + 1 + (int)(idx / cnt), j = p + 1 + (int)(idx % cnt);
            if (j >= i) W[(long long)i * ld + j] -= W[(long long)p * ld + i] * W[(long long)p * ld + j];
        }
        __syncthreads();
    }
    // Li = L^-1 with L = R^T (L[i][p] = W[p][i]): row p divided by L_pp, then row i -= L_ip row p for i > p
    for (long long idx = tid; idx < n2; idx += kCholThreads) Li[idx] = (idx / ld) == (idx % ld) ? 1.0 : 0.0;
    __syncthreads();
    for (int p = 0; p < ld; ++p) {
        const double d = 1.0 / W[(long long)p * ld + p];
        for (int j = tid; j <= p; j += kCholThreads) Li[(long long)p * ld + j] *= d;
        __syncthreads();
        const int cnt = ld - p - 1;
        for (long long idx = tid; idx < (long long)cnt * (p + 1); idx += kCholThreads) {
            const int i = p + 1 + (int)(idx / (p + 1)), j = (int)(idx % (p + 1));
            Li[(long long)i * ld + j] -= W[(long long)p * ld + i] * Li[(long long)p * ld + j];
        }
        __syncthreads();
    }
    if (!Racc) return;
    for (long long idx = tid; idx < n2; idx += kCholThreads) {
        const int i = (int)(idx / ld), j = (int)(idx % ld);
        double s = 0.0;
        if (j >= i) {
            if (racc_first) s = W[idx];
            else
                for (int k = i; k <= j; ++k) s += W[(long long)i * ld + k] * Racc[(long long)k * ld + j];
        }
        scratch[idx] = s;
    }
    __syncthreads();
    for (long long idx = tid; idx < n2; idx += kCholThreads) Racc[idx] = scratch[idx];
}

// out[tile rt, tile ct] = Y[rows of rt, :] R^-1[:, cols of ct] = sum_k Y[r, k] Li[c, k] over k < 64 (ct + 1) (Li lower)
__global__ void __launch_bounds__(256) psvd_apply_kernel(const double *__restrict__ Y, int ld, const double *__restrict__ Li,
                                                         double *__restrict__ out)
{
    __shared__ DmmaSmem sm;
    const int rt = blockIdx.x, ct = blockIdx.y;
    double acc[4][2][2] = {};
    dmma_nt_64(Y + (long long)rt * kDmmaTile * ld, ld, Li + (long long)ct * kDmmaTile * ld, ld, (ct + 1) * kDmmaTile, acc, sm);
#pragma unroll
    for (int mi = 0; mi < 4; ++mi)
#pragma unroll
        for (int ni = 0; ni < 2; ++ni)
#pragma unroll
            for (int e = 0; e < 2; ++e)
                out[(long long)(rt * kDmmaTile + dmma_row(mi)) * ld + ct * kDmmaTile + dmma_col(ni, e)] = acc[mi][ni][e];
}

struct OrthGeom {
    long long mp, chunk;
    int nchunks;
};

static OrthGeom orth_geom(long long m, int ld)
{
    OrthGeom g;
    g.mp = round_up(m, kDmmaTile);
    long long cap = (64ll << 20) / (8ll * ld * ld);
    long long n = (g.mp + 1023) / 1024;
    if (n > cap) n = cap;
    if (n < 1) n = 1;
    g.chunk = round_up((g.mp + n - 1) / n, kDmmaTile);
    g.nchunks = (int)((g.mp + g.chunk - 1) / g.chunk);
    return g;
}

struct OrthWs {
    int *flag;
    double *W, *Li, *scratch, *part, *tmp;
};

static size_t carve_orth(void *base, long long m, int ld, OrthWs *w)
{
    const OrthGeom g = orth_geom(m, ld);
    size_t off = 0;
    char *b = (char *)base;
    auto take = [&](size_t bytes) {
        char *p = b ? b + off : nullptr;
        off += (bytes + 255) & ~(size_t)255;
        return p;
    };
    const size_t sq = sizeof(double) * (size_t)ld * ld;
    OrthWs t;
    t.flag = (int *)take(256);
    t.W = (double *)take(sq);
    t.Li = (double *)take(sq);
    t.scratch = (double *)take(sq);
    t.part = (double *)take(sq * g.nchunks);
    t.tmp = (double *)take(sizeof(double) * (size_t)g.mp * ld);
    if (w) *w = t;
    return off;
}

// ---------------------------------------------------------------- small SVD
// One CTA.  A = R^T is kept by columns: row j of UT is column j of A (row j of R), row j of VT column j of V.  Round r of a
// sweep pairs (0, p_0) and (p_q, p_{L-1-q}), p_k = (k + r) mod (L - 1) + 1, L = l rounded up to even (index l: no pair).
__global__ void __launch_bounds__(kJacobiThreads) psvd_jacobi_kernel(const double *__restrict__ R, int l, int ld,
                                                                     double *__restrict__ UT, double *__restrict__ VT,
                                                                     double *__restrict__ s)
{
    __shared__ int s_rot;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = kJacobiThreads / 32;
    const long long n2 = (long long)ld * ld;
    for (long long idx = tid; idx < n2; idx += kJacobiThreads) {
        const int i = (int)(idx / ld), j = (int)(idx % ld);
        UT[idx] = i < l && j < l && j >= i ? R[idx] : 0.0;
        VT[idx] = i < l && i == j ? 1.0 : 0.0;
    }
    const int L = (l + 1) & ~1;
    // a pair is rotated while |a_p . a_q| > tol |a_p| |a_q|; the sweeps stop when no pair of a sweep exceeded l eps, the level
    // below which the computed dot product is rounding noise (a tighter stop can rotate on noise forever)
    const double tol = sqrt((double)l) * 2.0 * kUnit, stop = l * 2.0 * kUnit;
    for (int sweep = 0; sweep < kMaxSweeps; ++sweep) {
        if (tid == 0) s_rot = 0;
        __syncthreads();
        for (int r = 0; r < L - 1; ++r) {
            for (int q = warp; q < L / 2; q += nw) {
                int a = q == 0 ? 0 : (q + r) % (L - 1) + 1;
                int b = q == 0 ? r % (L - 1) + 1 : (L - 1 - q + r) % (L - 1) + 1;
                if (a > b) { const int x = a; a = b; b = x; }
                if (b >= l) continue;
                double *ap = UT + (long long)a * ld, *aq = UT + (long long)b * ld;
                double al = 0.0, be = 0.0, ga = 0.0;
                for (int c = lane; c < l; c += 32) {
                    const double x = ap[c], y = aq[c];
                    al = __fma_rn(x, x, al);
                    be = __fma_rn(y, y, be);
                    ga = __fma_rn(x, y, ga);
                }
                al = warp_sum(al);
                be = warp_sum(be);
                ga = warp_sum(ga);
                if (!(al > 0.0 && be > 0.0) || !(fabs(ga) > tol * sqrt(al) * sqrt(be))) continue;
                const bool big = fabs(ga) > stop * sqrt(al) * sqrt(be);
                const double zeta = (be - al) / (2.0 * ga);
                const double t = fabs(zeta) > 1e150 ? 0.5 / zeta : copysign(1.0, zeta) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
                const double cs = 1.0 / sqrt(1.0 + t * t), sn = cs * t;
                for (int c = lane; c < l; c += 32) {
                    const double x = ap[c], y = aq[c];
                    ap[c] = cs * x - sn * y;
                    aq[c] = sn * x + cs * y;
                }
                double *vp = VT + (long long)a * ld, *vq = VT + (long long)b * ld;
                for (int c = lane; c < l; c += 32) {
                    const double x = vp[c], y = vq[c];
                    vp[c] = cs * x - sn * y;
                    vq[c] = sn * x + cs * y;
                }
                if (lane == 0 && big) atomicAdd(&s_rot, 1);
            }
            __syncthreads();
        }
        const int rot = s_rot;
        __syncthreads();
        if (rot == 0) break;
    }
    for (int j = warp; j < l; j += nw) {
        double *aj = UT + (long long)j * ld;
        double ss = 0.0;
        for (int c = lane; c < l; c += 32) ss = __fma_rn(aj[c], aj[c], ss);
        const double sg = sqrt(warp_sum(ss));
        if (sg > 0.0)
            for (int c = lane; c < l; c += 32) aj[c] /= sg;
        if (lane == 0) s[j] = sg;
    }
}

// ---------------------------------------------------------------- factors
// perm[rank] = j by (sigma descending, index ascending); sorted[rank] = sigma_j
__global__ void psvd_sort_kernel(const double *__restrict__ s, int l, int *__restrict__ perm, double *__restrict__ sorted)
{
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < l; j += gridDim.x * blockDim.x) {
        int rank = 0;
        for (int i = 0; i < l; ++i) rank += s[i] > s[j] || (s[i] == s[j] && i < j);
        perm[rank] = j;
        sorted[rank] = s[j];
    }
}

// dst[c][:] = src[perm[c]][:] for c < k, 0 for k <= c < kp
__global__ void psvd_gather_rows_kernel(const double *__restrict__ src, const int *__restrict__ perm, int k, int kp, int ld,
                                        double *__restrict__ dst)
{
    const long long total = (long long)kp * ld;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(idx / ld), j = (int)(idx % ld);
        dst[idx] = c < k ? src[(long long)perm[c] * ld + j] : 0.0;
    }
}

// out [mp, kp] = P [mp, ld] . BT[kp, ld]^T on DMMA
__global__ void __launch_bounds__(256) psvd_mul_kernel(const double *__restrict__ P, int ld, const double *__restrict__ BT, int kp,
                                                       double *__restrict__ out)
{
    __shared__ DmmaSmem sm;
    const int rt = blockIdx.x, ct = blockIdx.y;
    double acc[4][2][2] = {};
    dmma_nt_64(P + (long long)rt * kDmmaTile * ld, ld, BT + (long long)ct * kDmmaTile * ld, ld, ld, acc, sm);
#pragma unroll
    for (int mi = 0; mi < 4; ++mi)
#pragma unroll
        for (int ni = 0; ni < 2; ++ni)
#pragma unroll
            for (int e = 0; e < 2; ++e)
                out[(long long)(rt * kDmmaTile + dmma_row(mi)) * kp + ct * kDmmaTile + dmma_col(ni, e)] = acc[mi][ni][e];
}

__device__ __forceinline__ bool amax_before(double va, long long ia, double vb, long long ib)
{
    return va > vb || (va == vb && ia < ib);
}

// a CTA per column c: the sign of the column's largest-magnitude entry over rows [0, rows), first index on ties
__global__ void __launch_bounds__(256) psvd_sign_kernel(const double *__restrict__ S, long long rows, int kp,
                                                        double *__restrict__ sign)
{
    __shared__ double wv[8];
    __shared__ long long wi[8];
    const int c = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double bv = -1.0;
    long long bi = 0x7fffffffffffffffll;
    for (long long r = threadIdx.x; r < rows; r += blockDim.x) {
        const double v = fabs(S[r * kp + c]);
        if (amax_before(v, r, bv, bi)) { bv = v; bi = r; }
    }
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, bv, off);
        const long long oi = __shfl_xor_sync(0xffffffffu, bi, off);
        if (amax_before(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
    if (lane == 0) { wv[warp] = bv; wi[warp] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 8; ++w)
            if (amax_before(wv[w], wi[w], bv, bi)) { bv = wv[w]; bi = wi[w]; }
        sign[c] = bi < rows && S[bi * kp + c] < 0.0 ? -1.0 : 1.0;
    }
}

// out[r][c] = (sign_c S[r][c]) (x sigma_c when given), c < k
__global__ void psvd_write_kernel(const double *__restrict__ S, long long rows, int kp, int k, const double *__restrict__ sign,
                                  const double *__restrict__ sigma, double *__restrict__ out)
{
    const long long total = rows * k;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const long long r = idx / k;
        const int c = (int)(idx % k);
        const double v = sign[c] * S[r * kp + c];
        out[idx] = sigma ? v * sigma[c] : v;
    }
}

struct FactorWs {
    int *perm;
    double *sign, *UkT, *VkT, *UA, *VA;
};

static size_t carve_factors(void *base, long long m, long long n, int ld, int k, FactorWs *w)
{
    const long long kp = round_up(k, kDmmaTile);
    size_t off = 0;
    char *b = (char *)base;
    auto take = [&](size_t bytes) {
        char *p = b ? b + off : nullptr;
        off += (bytes + 255) & ~(size_t)255;
        return p;
    };
    FactorWs t;
    t.perm = (int *)take(sizeof(int) * (size_t)ld);
    t.sign = (double *)take(sizeof(double) * (size_t)kp);
    t.UkT = (double *)take(sizeof(double) * (size_t)kp * ld);
    t.VkT = (double *)take(sizeof(double) * (size_t)kp * ld);
    t.UA = (double *)take(sizeof(double) * (size_t)round_up(m, kDmmaTile) * kp);
    t.VA = (double *)take(sizeof(double) * (size_t)round_up(n, kDmmaTile) * kp);
    if (w) *w = t;
    return off;
}

// ---------------------------------------------------------------- scoring
// warp per (row, candidate): user_vec[u] . item_vec[c], lanes over k in order, then the xor butterfly
__global__ void __launch_bounds__(256) psvd_scores_kernel(const double *__restrict__ P, const double *__restrict__ Qv, int k,
                                                          const int64_t *__restrict__ users, long long n,
                                                          const int64_t *__restrict__ cands, int C, double *__restrict__ out)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (long long row = blockIdx.y; row < n; row += gridDim.y) {
        const double *p = P + users[row] * k;
        for (long long c = (long long)blockIdx.x * 8 + warp; c < C; c += (long long)gridDim.x * 8) {
            const long long item = cands ? cands[row * C + c] : c;
            const double *q = Qv + item * k;
            double acc = 0.0;
            for (int j = lane; j < k; j += 32) acc = __fma_rn(p[j], q[j], acc);
            acc = warp_sum(acc);
            if (lane == 0) out[row * C + c] = acc;
        }
    }
}

}  // namespace drb

using namespace drb;

extern "C" int drb_puresvd_csr(const int64_t *d_seq_ptr, const int32_t *d_order, const int32_t *d_coo_i, const double *d_coo_v,
                               int32_t user_num, int32_t item_num, const int64_t *d_row_ptr, const int32_t *d_col, int64_t nnz,
                               const int64_t *d_t_ptr, const int32_t *d_t_col, double *d_val, double *d_t_val, void *stream)
{
    DRB_REQUIRE(d_seq_ptr && d_row_ptr && d_t_ptr && user_num > 0 && item_num > 0 && nnz >= 0 &&
                    (nnz == 0 || (d_order && d_coo_i && d_coo_v && d_col && d_t_col && d_val && d_t_val)),
                "puresvd_csr: bad arguments");
    if (nnz == 0) return DRB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    psvd_values_kernel<<<grid_for(user_num, 128), 128, 0, st>>>(d_seq_ptr, d_order, d_coo_i, d_coo_v, user_num, d_row_ptr, d_col,
                                                                 d_val);
    psvd_transpose_kernel<<<grid_for(nnz, 256), 256, 0, st>>>(d_row_ptr, d_col, d_val, d_t_ptr, d_t_col, item_num, nnz, d_t_val);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}

extern "C" int drb_puresvd_spmm(const int64_t *d_row_ptr, const int32_t *d_col, const double *d_val, int32_t n_rows,
                                const double *d_Z, int32_t l, int32_t ld, double *d_Y, void *stream)
{
    DRB_REQUIRE(d_row_ptr && d_Z && d_Y && n_rows >= 0 && l > 0 && ld >= l, "puresvd_spmm: bad arguments");
    if (n_rows == 0) return DRB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    for (int c0 = 0; c0 < ld; c0 += 32 * kSpmmCols) {
        const int nc = (ld - c0 + 31) / 32;
        switch (nc >= kSpmmCols ? kSpmmCols : nc) {
        case 1: spmm_launch<1>(d_row_ptr, d_col, d_val, n_rows, d_Z, ld, c0, l, d_Y, st); break;
        case 2: spmm_launch<2>(d_row_ptr, d_col, d_val, n_rows, d_Z, ld, c0, l, d_Y, st); break;
        case 3: spmm_launch<3>(d_row_ptr, d_col, d_val, n_rows, d_Z, ld, c0, l, d_Y, st); break;
        case 4: spmm_launch<4>(d_row_ptr, d_col, d_val, n_rows, d_Z, ld, c0, l, d_Y, st); break;
        case 5: spmm_launch<5>(d_row_ptr, d_col, d_val, n_rows, d_Z, ld, c0, l, d_Y, st); break;
        case 6: spmm_launch<6>(d_row_ptr, d_col, d_val, n_rows, d_Z, ld, c0, l, d_Y, st); break;
        case 7: spmm_launch<7>(d_row_ptr, d_col, d_val, n_rows, d_Z, ld, c0, l, d_Y, st); break;
        default: spmm_launch<8>(d_row_ptr, d_col, d_val, n_rows, d_Z, ld, c0, l, d_Y, st); break;
        }
    }
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}

extern "C" size_t drb_puresvd_orth_workspace_bytes(int64_t m, int32_t ld)
{
    if (m <= 0 || ld <= 0 || ld % kDmmaTile) return 0;
    return carve_orth(nullptr, m, ld, nullptr);
}

extern "C" int drb_puresvd_orth(double *d_Y, int64_t m, int32_t l, int32_t ld, void *d_ws, double *d_R, void *stream)
{
    DRB_REQUIRE(d_Y && d_ws && m > 0 && l > 0 && l <= 1024 && ld == round_up(l, kDmmaTile), "puresvd_orth: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    OrthWs w;
    carve_orth(d_ws, m, ld, &w);
    const OrthGeom g = orth_geom(m, ld);
    const int T = ld / kDmmaTile;
    DRB_REQUIRE(g.mp / kDmmaTile < (1ll << 31), "puresvd_orth: %lld rows exceed the tile grid", (long long)m);
    const long long n2 = (long long)ld * ld;
    DRB_CUDA(cudaMemsetAsync(w.flag, 0, sizeof(int), st));
    double *src = d_Y, *dst = w.tmp;
    for (int pass = 0; pass < 3; ++pass) {
        psvd_gram_kernel<<<dim3(T, T, g.nchunks), 256, 0, st>>>(src, g.mp, ld, g.chunk, w.part);
        psvd_gram_reduce_kernel<<<grid_for(n2, 256), 256, 0, st>>>(w.part, g.nchunks, n2, w.W);
        psvd_chol_kernel<<<1, kCholThreads, 0, st>>>(w.W, l, ld, m, pass == 0, w.Li, d_R, pass == 0, w.scratch, w.flag);
        psvd_apply_kernel<<<dim3((unsigned)(g.mp / kDmmaTile), T), 256, 0, st>>>(src, ld, w.Li, dst);
        DRB_CUDA(cudaGetLastError());
        double *x = src; src = dst; dst = x;
    }
    DRB_CUDA(cudaMemcpyAsync(d_Y, src, sizeof(double) * (size_t)g.mp * ld, cudaMemcpyDeviceToDevice, st));
    int flag = 0;
    DRB_CUDA(cudaMemcpyAsync(&flag, w.flag, sizeof(int), cudaMemcpyDeviceToHost, st));
    DRB_CUDA(cudaStreamSynchronize(st));
    if (flag) {
        set_error("puresvd_orth: the panel is numerically rank deficient (a Cholesky pivot <= l u max diag)");
        return DRB_ERR_NOT_PD;
    }
    return DRB_OK;
}

extern "C" int drb_puresvd_small_svd(const double *d_R, int32_t l, int32_t ld, double *d_s, double *d_UT, double *d_VT,
                                     void *stream)
{
    DRB_REQUIRE(d_R && d_s && d_UT && d_VT && l > 0 && l <= 1024 && ld >= l, "puresvd_small_svd: bad arguments");
    psvd_jacobi_kernel<<<1, kJacobiThreads, 0, (cudaStream_t)stream>>>(d_R, l, ld, d_UT, d_VT, d_s);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}

extern "C" size_t drb_puresvd_factors_workspace_bytes(int64_t m, int64_t n, int32_t ld, int32_t k)
{
    if (m <= 0 || n <= 0 || ld <= 0 || k <= 0) return 0;
    return carve_factors(nullptr, m, n, ld, k, nullptr);
}

extern "C" int drb_puresvd_factors(const double *d_Q, int64_t m, const double *d_Qb, int64_t n, int32_t l, int32_t ld,
                                   const double *d_s, const double *d_UT, const double *d_VT, int32_t transposed, int32_t k,
                                   void *d_ws, double *d_user_vec, double *d_item_vec, double *d_sigma, void *stream)
{
    DRB_REQUIRE(d_Q && d_Qb && d_s && d_UT && d_VT && d_ws && d_user_vec && d_item_vec && d_sigma && m > 0 && n > 0 && l > 0 &&
                    ld == round_up(l, kDmmaTile) && k > 0 && k <= l,
                "puresvd_factors: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    FactorWs w;
    carve_factors(d_ws, m, n, ld, k, &w);
    const int kp = (int)round_up(k, kDmmaTile);
    psvd_sort_kernel<<<(l + 255) / 256, 256, 0, st>>>(d_s, l, w.perm, d_sigma);
    psvd_gather_rows_kernel<<<grid_for((long long)kp * ld, 256), 256, 0, st>>>(d_UT, w.perm, k, kp, ld, w.UkT);
    psvd_gather_rows_kernel<<<grid_for((long long)kp * ld, 256), 256, 0, st>>>(d_VT, w.perm, k, kp, ld, w.VkT);
    psvd_mul_kernel<<<dim3((unsigned)(round_up(m, kDmmaTile) / kDmmaTile), kp / kDmmaTile), 256, 0, st>>>(d_Q, ld, w.UkT, kp, w.UA);
    psvd_mul_kernel<<<dim3((unsigned)(round_up(n, kDmmaTile) / kDmmaTile), kp / kDmmaTile), 256, 0, st>>>(d_Qb, ld, w.VkT, kp, w.VA);
    // the user side: U_A (rows of X) when A = X, V_A (columns of X^T) when A = X^T
    const double *user = transposed ? w.VA : w.UA, *item = transposed ? w.UA : w.VA;
    const long long un = transposed ? n : m, in = transposed ? m : n;
    psvd_sign_kernel<<<k, 256, 0, st>>>(user, un, kp, w.sign);
    psvd_write_kernel<<<grid_for(un * k, 256), 256, 0, st>>>(user, un, kp, k, w.sign, nullptr, d_user_vec);
    psvd_write_kernel<<<grid_for(in * k, 256), 256, 0, st>>>(item, in, kp, k, w.sign, d_sigma, d_item_vec);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}

extern "C" int drb_puresvd_scores(const double *d_user_vec, const double *d_item_vec, int32_t k, const int64_t *d_users,
                                  int64_t n_users, const int64_t *d_cands, int32_t cand_num, double *d_scores, void *stream)
{
    DRB_REQUIRE(d_user_vec && d_item_vec && d_users && d_scores && k > 0 && n_users >= 0 && cand_num > 0,
                "puresvd_scores: bad arguments");
    if (n_users == 0) return DRB_OK;
    const unsigned gy = (unsigned)(n_users < 65535 ? n_users : 65535);
    const unsigned gx = (unsigned)((cand_num + 7) / 8 < 1024 ? (cand_num + 7) / 8 : 1024);
    psvd_scores_kernel<<<dim3(gx, gy), 256, 0, (cudaStream_t)stream>>>(d_user_vec, d_item_vec, k, d_users, n_users, d_cands,
                                                                       cand_num, d_scores);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}
