// neumf_fused.cuh -- the whole NeuMF tower step of a 64-triple tile inside ONE CTA: activations never leave the SM.
//
// Stands behind NeuMF.forward / calc_loss / backward (daisy/model/NeuMFRecommender.py:118-169) for model_name 'NeuMF',
// num_layers = 2, factors = 32, dropout 0 (BASELINE config 3: F = 32, tower 128 -> 64 -> 32).  The layer-wise
// path (neumf.cu: gather, 2 forward GEMMs, head, 4 backward GEMMs, 2 column sums, scatter) streams fp32 activations through
// HBM between ~12 launches.  Here one persistent CTA per SM (four warpgroups) walks tiles of 64 triples = 128 rows
// (rows 0..63 the pos items, 64..127 the neg items of the same triples):
//
//   gather   A0 = cat(UM[u], IM[item]) rounded to bf16 straight into the K-major core-matrix image the tensor core reads
//            (lane group per row, 128-bit loads; the user row is loaded once and stored for both of its tile rows)
//   MMA      Z1 = A0 W1^T                      wgmma m64nNk16 bf16, fp32 accumulators in registers
//   epilogue A1 = relu(Z1 + b1) -> bf16 image (straight from the accumulator fragment)
//   MMA      Z2 = A1 W2^T
//   head     h = relu(Z2 + b2);  pred = wp . cat(UG[u] * IG[item], h) + bp;  x = pred_pos - pred_neg (rows r and r + 64 meet
//            through shared memory);  c = BPR coefficient;  loss / regulariser norms;  GMF-table gradients by RED;
//            dZ2 = +-c wp_h [h > 0] -> bf16 image
//   MMA      dA1 = dZ2 W2;   gW2^T += A1^T dZ2  (register accumulators carried over ALL tiles of the CTA)
//   epilogue dZ1 = dA1 [A1 > 0] -> bf16 image
//   MMA      dA0 = dZ1 W1;   gW1^T += A0^T dZ1  (carried over all tiles)
//   epilogue dA0 -> RED.128 into gUM[u] / gIM[item]
//   finally  the two weight gradients leave the registers once per CTA; bias / predict-layer gradients, loss and norms are
//            carried in registers across tiles and reduced once.
// Every product is split over the four warpgroups: warpgroup g takes row half (g & 1) -- or, for the A^T dZ products, K half
// or feature half -- and column half (g >> 1), so each issues m64n32 / m64n16 MMAs on its own accumulators.
// Every activation / gradient tile is written ONCE as a K-major operand image (element (row, k) at
// (k/8) LBO + (row/8) 128 + (row%8) 16 + (k%8) 2).  The same bytes are the MN-major image of the TRANSPOSED tile when the
// descriptor's two strides are swapped (K-group stride 128, MN-group stride LBO), which is how A^T dZ and dZ W are fed
// without a second copy.  HBM traffic per triple: the gather and scatter of the 96-float rows (2.3 KB, SURVEY 8(d)).
#pragma once
#include "umma_gemm.cuh"

namespace drb {

constexpr int kFusedThreads = 512;      // 4 warpgroups: row (or K / feature) half = g & 1, column half = g >> 1
constexpr int kFusedTile = 64;          // triples per tile (128 rows)

struct FusedParams {
    const float *UG, *IG, *UM, *IM;     // tables
    const float *W;                     // tower block: W1 [N1, N0], b1 [N1], W2 [N2, N1], b2 [N2], wp [2F], bp
    const int32_t *bu, *bi, *bj;
    long long B;                        // triples in this step
    float *gUG, *gIG, *gUM, *gIM, *gW;  // gradient accumulators (table-shaped; gW like W)
    unsigned *cntU;
    unsigned long long *cntI;
    double *red;                        // [11] bpr, l1[5], s2[5]  (UG_u, UM_u, IG_i, IM_i, IG_j)
    int has_reg, apply;
};

__host__ __device__ constexpr uint32_t fused_lbo(int rows) { return (uint32_t)(rows / 8) * 128u + 32u; }

template <int F>
struct FusedLayout {
    static constexpr int D = 2 * F, N0 = 4 * F, N1 = 2 * F, N2 = F;
    static constexpr uint32_t LBO_T = fused_lbo(128);                 // images with 128 tile rows
    static constexpr uint32_t LBO_W1 = fused_lbo(N1), LBO_W2 = fused_lbo(N2);
    static constexpr uint32_t A0 = 0;
    static constexpr uint32_t A1 = A0 + (N0 / 8) * LBO_T;
    static constexpr uint32_t DZ1 = A1 + (N1 / 8) * LBO_T;
    static constexpr uint32_t DZ2 = DZ1 + (N1 / 8) * LBO_T;
    static constexpr uint32_t W1 = DZ2 + (N2 / 8) * LBO_T;
    static constexpr uint32_t W2 = W1 + (N0 / 8) * LBO_W1;
    static constexpr uint32_t W_END = W2 + (N1 / 8) * LBO_W2;
    // fp32 staging of the NEXT tile's gathered rows (cp.async): MLP rows [3][64][D], GMF rows [3][64][F + 4] (padded)
    static constexpr uint32_t SM = (W_END + 127) / 128 * 128;
    static constexpr uint32_t SG = SM + 3 * 64 * D * 4;
    static constexpr int GROW = F + 4;
    static constexpr uint32_t TAIL = SG + 3 * 64 * GROW * 4;
    static constexpr uint32_t BYTES = (TAIL + 127) / 128 * 128;
};

// bf16 pair (k, k + 1), k even, of tile row `row` of a K-major image with 128 rows: one 4-byte store
__device__ __forceinline__ uint32_t image_off(uint32_t lbo, int row, int k)
{
    return (uint32_t)(k >> 3) * lbo + (uint32_t)(row >> 3) * 128u + (uint32_t)(row & 7) * 16u + (uint32_t)(k & 7) * 2u;
}
__device__ __forceinline__ void image_store2(unsigned char *img, uint32_t lbo, int row, int k, float a, float b)
{
    *reinterpret_cast<uint32_t *>(img + image_off(lbo, row, k)) = pack_bf16x2(a, b);
}
__device__ __forceinline__ bool bf16_positive(uint32_t hbits) { return (hbits & 0x7fffu) != 0u && (hbits & 0x8000u) == 0u; }

template <int F>
__global__ void __launch_bounds__(kFusedThreads, 1) neumf_fused_kernel(FusedParams p)
{
    using L = FusedLayout<F>;
    constexpr int D = L::D, N0 = L::N0, N1 = L::N1, N2 = L::N2;
    static_assert(N0 == 128 && N1 == 64 && N2 == 32, "the warpgroup split is written for factors = 32");
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ float s_b1[N1], s_b2[N2], s_wp[2 * F + 1];
    __shared__ float s_pred[2][128];
    __shared__ int s_idx[2][3][kFusedTile];       // [buffer][u | i | j][triple] of the current and the next tile
    __shared__ float s_colsum[N1 + N2 + 2 * F];   // final cross-thread reduction of the register column sums
    __shared__ double s_red[11];

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int wg = tid >> 7, mh = wg & 1, nh = wg >> 1;     // row (K, feature) half and column half of this warpgroup
    const int quad = lane & 3;
    const int rbase = mh * 64 + (warp & 3) * 16 + (lane >> 2);   // fragment rows rbase and rbase + 8
    const bool pos_row = mh == 0;                            // rows 0..63: pos items, 64..127: neg items
    const float sign = pos_row ? 1.f : -1.f;

    // ---- one-off: weights as bf16 operand images, biases
    const float *W1 = p.W, *b1 = W1 + (size_t)N1 * N0, *W2 = b1 + N1, *b2 = W2 + (size_t)N2 * N1, *wp = b2 + N2;
    for (int it = tid; it < N1 * (N0 / 8); it += kFusedThreads) {            // W1 [N1 rows, N0 k] K-major image
        const int r = it / (N0 / 8), kg = it % (N0 / 8);
        const float4 *s4 = reinterpret_cast<const float4 *>(W1 + (size_t)r * N0 + kg * 8);
        const float4 a = __ldg(s4), b = __ldg(s4 + 1);
        uint4 o;
        o.x = pack_bf16x2(a.x, a.y); o.y = pack_bf16x2(a.z, a.w); o.z = pack_bf16x2(b.x, b.y); o.w = pack_bf16x2(b.z, b.w);
        *reinterpret_cast<uint4 *>(smem + L::W1 + (uint32_t)kg * L::LBO_W1 + (uint32_t)(r >> 3) * 128u + (uint32_t)(r & 7) * 16u) = o;
    }
    for (int it = tid; it < N2 * (N1 / 8); it += kFusedThreads) {            // W2 [N2 rows, N1 k]
        const int r = it / (N1 / 8), kg = it % (N1 / 8);
        const float4 *s4 = reinterpret_cast<const float4 *>(W2 + (size_t)r * N1 + kg * 8);
        const float4 a = __ldg(s4), b = __ldg(s4 + 1);
        uint4 o;
        o.x = pack_bf16x2(a.x, a.y); o.y = pack_bf16x2(a.z, a.w); o.z = pack_bf16x2(b.x, b.y); o.w = pack_bf16x2(b.z, b.w);
        *reinterpret_cast<uint4 *>(smem + L::W2 + (uint32_t)kg * L::LBO_W2 + (uint32_t)(r >> 3) * 128u + (uint32_t)(r & 7) * 16u) = o;
    }
    for (int k = tid; k < N1; k += kFusedThreads) s_b1[k] = b1[k];
    for (int k = tid; k < N2; k += kFusedThreads) s_b2[k] = b2[k];
    for (int k = tid; k < 2 * F + 1; k += kFusedThreads) s_wp[k] = wp[k];
    if (tid < 11) s_red[tid] = 0.0;
    for (int k = tid; k < N1 + N2 + 2 * F; k += kFusedThreads) s_colsum[k] = 0.f;
    __syncthreads();
    const uint32_t sbase = smem_u32(smem);

    // register accumulators carried across tiles (reduced once at the end)
    float acc_loss = 0.f, acc_l1[5] = {0, 0, 0, 0, 0}, acc_s2[5] = {0, 0, 0, 0, 0};
    float gw1[16], gw2[8];                        // gW1^T [features of half mh] x [outputs of half nh]; gW2^T K-half mh
    float gb1[8], gb2[4], gwg[4], gwh[4];         // column sums of this thread's fragment columns
#pragma unroll
    for (int k = 0; k < 16; ++k) gw1[k] = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) { gw2[k] = 0.f; gb1[k] = 0.f; }
#pragma unroll
    for (int k = 0; k < 4; ++k) { gb2[k] = 0.f; gwg[k] = 0.f; gwh[k] = 0.f; }

    const long long ntiles = (p.B + kFusedTile - 1) / kFusedTile;
    bool first_tile = true;

    // a tile's index lists: threads 0..191 hold one index each (u | i | j of triple tid % 64)
    auto fetch_index = [&](long long tile_) {
        int v = 0;
        if (tid < 3 * kFusedTile) {
            const int kind = tid / kFusedTile, r = tid % kFusedTile;
            const long long t = tile_ * kFusedTile + r;
            if (t < p.B) v = __ldg((kind == 0 ? p.bu : kind == 1 ? p.bi : p.bj) + t);
        }
        return v;
    };
    auto store_index = [&](int v, int buf) {
        if (tid < 3 * kFusedTile) s_idx[buf][tid / kFusedTile][tid % kFusedTile] = v;
    };
    // asynchronous global -> shared copies (cp.async, 16 bytes per lane) of a tile's gathered rows, straight from the tables
    constexpr int G = D / 4;                               // lanes per D-float MLP row
    constexpr int GROUPS = kFusedThreads / G;
    constexpr int GG = F / 4;                              // lanes per F-float GMF row
    constexpr int GGROUPS = kFusedThreads / GG;
    auto prefetch_mlp = [&](long long tile_, int buf) {
        const int nt_ = (int)min((long long)kFusedTile, p.B - tile_ * kFusedTile);
        const int gl = tid % G, grp = tid / G;
#pragma unroll
        for (int w = grp; w < 3 * kFusedTile; w += GROUPS) {
            const int kind = w / kFusedTile, r = w % kFusedTile;            // 0: UM[u], 1: IM[i], 2: IM[j]
            const uint32_t off = L::SM + (uint32_t)(w * D + gl * 4) * 4u;
            if (r < nt_) {
                const float *src = (kind == 0 ? p.UM : p.IM) + (size_t)s_idx[buf][kind][r] * D + gl * 4;
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sbase + off), "l"(src) : "memory");
            } else {
                *reinterpret_cast<float4 *>(smem + off) = make_float4(0.f, 0.f, 0.f, 0.f);
            }
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    auto prefetch_gmf = [&](long long tile_, int buf) {
        const int nt_ = (int)min((long long)kFusedTile, p.B - tile_ * kFusedTile);
        const int gl = tid % GG, grp = tid / GG;
#pragma unroll
        for (int w = grp; w < 3 * kFusedTile; w += GGROUPS) {
            const int kind = w / kFusedTile, r = w % kFusedTile;            // 0: UG[u], 1: IG[i], 2: IG[j]
            const uint32_t off = L::SG + (uint32_t)(w * L::GROW + gl * 4) * 4u;
            if (r < nt_) {
                const float *src = (kind == 0 ? p.UG : p.IG) + (size_t)s_idx[buf][kind][r] * F + gl * 4;
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sbase + off), "l"(src) : "memory");
            } else {
                *reinterpret_cast<float4 *>(smem + off) = make_float4(0.f, 0.f, 0.f, 0.f);
            }
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    int cur = 0;
    if ((long long)blockIdx.x < ntiles) {
        store_index(fetch_index(blockIdx.x), 0);
        __syncthreads();
        prefetch_mlp(blockIdx.x, 0);
        prefetch_gmf(blockIdx.x, 0);
    }
    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x, cur ^= 1) {
        const long long t0 = tile * kFusedTile;
        const int nt = (int)min((long long)kFusedTile, p.B - t0);           // valid triples in this tile
        const long long next_tile = tile + gridDim.x;
        const bool has_next = next_tile < ntiles;
        const int idx_next = has_next ? fetch_index(next_tile) : 0;        // lands while this tile's rows are converted
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncthreads();                                                    // staged rows of this tile visible to everyone
        int trr[2], uu[2], itm[2];
        bool ok[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            trr[i] = (rbase + 8 * i) & (kFusedTile - 1);                    // triple of fragment row i
            ok[i] = trr[i] < nt;
            uu[i] = s_idx[cur][0][trr[i]];
            itm[i] = s_idx[cur][pos_row ? 1 : 2][trr[i]];
        }

        // ---------------------------------------------------------------- A0: staged fp32 rows -> bf16 K-major image
        {
            const int gl = tid % G, grp = tid / G;
#pragma unroll
            for (int w = grp; w < 3 * kFusedTile; w += GROUPS) {
                const int kind = w / kFusedTile, r = w % kFusedTile;        // 0: UM[u] -> rows r and r+64; 1: IM[i]; 2: IM[j]
                const float4 v = *reinterpret_cast<const float4 *>(smem + L::SM + (uint32_t)(w * D + gl * 4) * 4u);
                if (p.has_reg && kind < 2 && r < nt) {     // UM_u and IM_i rows enter the regulariser once per triple
                    const float a = fabsf(v.x) + fabsf(v.y) + fabsf(v.z) + fabsf(v.w);
                    const float s2 = fmaf(v.x, v.x, fmaf(v.y, v.y, fmaf(v.z, v.z, v.w * v.w)));
                    if (kind == 0) { acc_l1[1] += a; acc_s2[1] += s2; } else { acc_l1[3] += a; acc_s2[3] += s2; }
                }
                uint2 o;
                o.x = pack_bf16x2(v.x, v.y);
                o.y = pack_bf16x2(v.z, v.w);
                const int k = (kind == 0 ? 0 : D) + gl * 4;
                const int trow = kind == 2 ? r + kFusedTile : r;
                const uint32_t off = L::A0 + image_off(L::LBO_T, trow, k);
                *reinterpret_cast<uint2 *>(smem + off) = o;
                if (kind == 0) *reinterpret_cast<uint2 *>(smem + off + (kFusedTile >> 3) * 128u) = o;   // the neg row of the triple
            }
        }
        if (has_next) store_index(idx_next, cur ^ 1);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();

        // ---------------------------------------------------------------- Z1 = A0 W1^T  (rows of half mh, columns of half nh)
        float z1[16];
#pragma unroll
        for (int e = 0; e < 16; ++e) z1[e] = 0.f;
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < N0 / 16; ++kk)
            wgmma_m64n32<0, 0>(z1, umma_smem_desc(sbase + L::A0 + mh * 1024 + kk * 2 * L::LBO_T, L::LBO_T, 128),
                               umma_smem_desc(sbase + L::W1 + nh * 512 + kk * 2 * L::LBO_W1, L::LBO_W1, 128), kk > 0);
        wgmma_commit();
        if (has_next) prefetch_mlp(next_tile, cur ^ 1);      // the MLP staging has been consumed: refill it under the MMAs
        wgmma_wait_all();
        wgmma_fence_operand(z1);

        // ---------------------------------------------------------------- A1 = relu(Z1 + b1) -> image
#pragma unroll
        for (int nb = 0; nb < 4; ++nb) {
            const int col = nh * 32 + nb * 8 + 2 * quad;
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const float za = z1[nb * 4 + 2 * i] + s_b1[col], zb = z1[nb * 4 + 2 * i + 1] + s_b1[col + 1];
                image_store2(smem + L::A1, L::LBO_T, rbase + 8 * i, col, (ok[i] && za > 0.f) ? za : 0.f,
                             (ok[i] && zb > 0.f) ? zb : 0.f);
            }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();

        // ---------------------------------------------------------------- Z2 = A1 W2^T  (rows of half mh, 16 columns of half nh)
        float z2[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) z2[e] = 0.f;
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < N1 / 16; ++kk)
            wgmma_m64n16<0, 0>(z2, umma_smem_desc(sbase + L::A1 + mh * 1024 + kk * 2 * L::LBO_T, L::LBO_T, 128),
                               umma_smem_desc(sbase + L::W2 + nh * 256 + kk * 2 * L::LBO_W2, L::LBO_W2, 128), kk > 0);
        wgmma_commit();
        // GMF rows at this thread's columns 16 nh + 8 nb + 2 quad + {0, 1} (rows beyond the batch were staged as zeros)
        float gu[2][4], gi[2][4];
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int nb = 0; nb < 2; ++nb) {
                const int col = nh * 16 + nb * 8 + 2 * quad;
                const float2 a = *reinterpret_cast<const float2 *>(smem + L::SG + (uint32_t)((0 * kFusedTile + trr[i]) * L::GROW + col) * 4u);
                const float2 b = *reinterpret_cast<const float2 *>(
                    smem + L::SG + (uint32_t)(((pos_row ? 1 : 2) * kFusedTile + trr[i]) * L::GROW + col) * 4u);
                gu[i][2 * nb] = a.x; gu[i][2 * nb + 1] = a.y;
                gi[i][2 * nb] = b.x; gi[i][2 * nb + 1] = b.y;
            }
        wgmma_wait_all();
        wgmma_fence_operand(z2);

        // ---------------------------------------------------------------- head: h, prediction, BPR coefficient, dZ2, GMF gradients
        float hval[2][4];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            float part_sum = 0.f;
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int col = nh * 16 + (e >> 1) * 8 + 2 * quad + (e & 1);
                const float z = z2[(e >> 1) * 4 + 2 * i + (e & 1)] + s_b2[col];
                hval[i][e] = (ok[i] && z > 0.f) ? z : 0.f;
                part_sum = fmaf(s_wp[F + col], hval[i][e], part_sum);
                part_sum = fmaf(s_wp[col], gu[i][e] * gi[i][e], part_sum);
            }
            part_sum += __shfl_xor_sync(0xffffffffu, part_sum, 1);
            part_sum += __shfl_xor_sync(0xffffffffu, part_sum, 2);
            if (quad == 0) s_pred[nh][rbase + 8 * i] = part_sum;
            if (p.has_reg && ok[i]) {
                float a1 = 0.f, q1 = 0.f, a2 = 0.f, q2 = 0.f;
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    a1 += fabsf(gu[i][e]); q1 = fmaf(gu[i][e], gu[i][e], q1);
                    a2 += fabsf(gi[i][e]); q2 = fmaf(gi[i][e], gi[i][e], q2);
                }
                if (pos_row) { acc_l1[0] += a1; acc_s2[0] += q1; acc_l1[2] += a2; acc_s2[2] += q2; }   // UG_u once, IG_i
                else { acc_l1[4] += a2; acc_s2[4] += q2; }                                               // IG_j
            }
        }
        __syncthreads();
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int tr = trr[i];
            const float pp = s_pred[0][tr] + s_pred[1][tr];
            const float pn = s_pred[0][tr + kFusedTile] + s_pred[1][tr + kFusedTile];
            const float x = pp - pn;                                    // the predict bias cancels in the pair
            const float sg = 1.f / (1.f + expf(-x));
            if (ok[i] && pos_row && nh == 0 && quad == 0) acc_loss += -logf(1e-10f + sg);
            const float cbpr = -(sg * (1.f - sg)) / (1e-10f + sg);
            const float dp = ok[i] ? sign * cbpr : 0.f;                 // d loss / d pred of THIS row
            float dz[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int col = nh * 16 + (e >> 1) * 8 + 2 * quad + (e & 1);
                dz[e] = hval[i][e] > 0.f ? dp * s_wp[F + col] : 0.f;
                gb2[e] += dz[e];
                gwh[e] += dp * hval[i][e];
                gwg[e] += dp * (gu[i][e] * gi[i][e]);
            }
            image_store2(smem + L::DZ2, L::LBO_T, rbase + 8 * i, nh * 16 + 2 * quad, dz[0], dz[1]);
            image_store2(smem + L::DZ2, L::LBO_T, rbase + 8 * i, nh * 16 + 8 + 2 * quad, dz[2], dz[3]);
            if (p.apply && ok[i]) {
#pragma unroll
                for (int nb = 0; nb < 2; ++nb) {
                    const int col = nh * 16 + nb * 8 + 2 * quad;
                    const float w0 = dp * s_wp[col], w1 = dp * s_wp[col + 1];
                    Vec<2> g1, g2;
                    g1.v[0] = w0 * gi[i][2 * nb]; g1.v[1] = w1 * gi[i][2 * nb + 1];     // d / d UG[u]
                    g2.v[0] = w0 * gu[i][2 * nb]; g2.v[1] = w1 * gu[i][2 * nb + 1];     // d / d IG[item]
                    red_row<2>(p.gUG + (size_t)uu[i] * F + col, g1);
                    red_row<2>(p.gIG + (size_t)itm[i] * F + col, g2);
                }
                if (nh == 0 && quad == 0) {
                    if (pos_row) {
                        red_add_u32(p.cntU + uu[i], 1u);
                        red_add_u64(p.cntI + itm[i], 1ull);
                    } else {
                        red_add_u64(p.cntI + itm[i], 1ull << 32);
                    }
                }
            }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
        if (!p.apply) {                                      // loss only
            if (has_next) prefetch_gmf(next_tile, cur ^ 1);
            first_tile = false;
            continue;
        }

        // ---------------------------------------------------------------- dA1 = dZ2 W2 ;  gW2^T += A1^T dZ2
        float da1[16];
#pragma unroll
        for (int e = 0; e < 16; ++e) da1[e] = 0.f;
        wgmma_fence();
        // B = W2 read transposed (MN-major view of its K-major image): mn = in (N1), k = out (N2)
#pragma unroll
        for (int kk = 0; kk < N2 / 16; ++kk)
            wgmma_m64n32<0, 1>(da1, umma_smem_desc(sbase + L::DZ2 + mh * 1024 + kk * 2 * L::LBO_T, L::LBO_T, 128),
                               umma_smem_desc(sbase + L::W2 + nh * 4 * L::LBO_W2 + kk * 256, 128, L::LBO_W2), kk > 0);
        // A = A1^T (features on the M side, tile rows of half mh as K), B = dZ2 read transposed: both MN-major views
#pragma unroll
        for (int kk = 0; kk < 64 / 16; ++kk)
            wgmma_m64n16<1, 1>(gw2, umma_smem_desc(sbase + L::A1 + mh * 1024 + kk * 256, 128, L::LBO_T),
                               umma_smem_desc(sbase + L::DZ2 + nh * 2 * L::LBO_T + mh * 1024 + kk * 256, 128, L::LBO_T), 1u);
        wgmma_commit();
        if (has_next) prefetch_gmf(next_tile, cur ^ 1);      // the GMF staging has been consumed by the head
        wgmma_wait_all();
        wgmma_fence_operand(da1);
        wgmma_fence_operand(gw2);

        // ---------------------------------------------------------------- dZ1 = dA1 [A1 > 0] -> image
#pragma unroll
        for (int nb = 0; nb < 4; ++nb) {
            const int col = nh * 32 + nb * 8 + 2 * quad;
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const uint32_t mw = *reinterpret_cast<const uint32_t *>(smem + L::A1 + image_off(L::LBO_T, rbase + 8 * i, col));
                const float va = bf16_positive(mw & 0xffffu) ? da1[nb * 4 + 2 * i] : 0.f;
                const float vb = bf16_positive(mw >> 16) ? da1[nb * 4 + 2 * i + 1] : 0.f;
                gb1[2 * nb] += va;
                gb1[2 * nb + 1] += vb;
                image_store2(smem + L::DZ1, L::LBO_T, rbase + 8 * i, col, va, vb);
            }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();

        // ---------------------------------------------------------------- dA0 = dZ1 W1 ;  gW1^T += A0^T dZ1
        float da0[2][16];
#pragma unroll
        for (int s = 0; s < 2; ++s)
#pragma unroll
            for (int e = 0; e < 16; ++e) da0[s][e] = 0.f;
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < N1 / 16; ++kk) {
            const uint64_t da = umma_smem_desc(sbase + L::DZ1 + mh * 1024 + kk * 2 * L::LBO_T, L::LBO_T, 128);
#pragma unroll
            for (int s = 0; s < 2; ++s)
                wgmma_m64n32<0, 1>(da0[s], da, umma_smem_desc(sbase + L::W1 + (nh * 8 + s * 4) * L::LBO_W1 + kk * 256, 128, L::LBO_W1),
                                   kk > 0);
        }
#pragma unroll
        for (int kk = 0; kk < 128 / 16; ++kk)
            wgmma_m64n32<1, 1>(gw1, umma_smem_desc(sbase + L::A0 + mh * 8 * L::LBO_T + kk * 256, 128, L::LBO_T),
                               umma_smem_desc(sbase + L::DZ1 + nh * 4 * L::LBO_T + kk * 256, 128, L::LBO_T), 1u);
        wgmma_commit();
        wgmma_wait_all();
        wgmma_fence_operand(da0[0]);
        wgmma_fence_operand(da0[1]);
        wgmma_fence_operand(gw1);

        // ---------------------------------------------------------------- scatter dA0: column half 0 -> gUM[u], half 1 -> gIM[item]
        // lanes 2j and 2j+1 swap half their pairs, so each lane holds 4 consecutive columns of one row: one RED.128 each
        {
            const int odd = lane & 1;
            float *dst = nh == 0 ? p.gUM + (size_t)uu[odd] * D : p.gIM + (size_t)itm[odd] * D;
#pragma unroll
            for (int s = 0; s < 2; ++s)
#pragma unroll
                for (int nb = 0; nb < 4; ++nb) {
                    const float *d4 = &da0[s][nb * 4];
                    const float s0 = odd ? d4[0] : d4[2], s1 = odd ? d4[1] : d4[3];
                    const float r0 = __shfl_xor_sync(0xffffffffu, s0, 1), r1 = __shfl_xor_sync(0xffffffffu, s1, 1);
                    Vec<4> g;
                    if (odd) { g.v[0] = r0; g.v[1] = r1; g.v[2] = d4[2]; g.v[3] = d4[3]; }
                    else { g.v[0] = d4[0]; g.v[1] = d4[1]; g.v[2] = r0; g.v[3] = r1; }
                    if (ok[odd]) red_row<4>(dst + s * 32 + nb * 8 + 2 * (quad & 2), g);
                }
        }
        first_tile = false;
        __syncthreads();                                     // images free for the next tile
    }

    // ---------------------------------------------------------------- once per CTA: weight gradients out of the registers
    if (p.apply && !first_tile) {
        float *gW1 = p.gW, *gb1g = gW1 + (size_t)N1 * N0, *gW2 = gb1g + N1, *gb2g = gW2 + (size_t)N2 * N1, *gwp = gb2g + N2;
#pragma unroll
        for (int nb = 0; nb < 4; ++nb)
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int c = 0; c < 2; ++c)      // gW1^T: row = input feature m, column = output n
                    atomicAdd(gW1 + (size_t)(nh * 32 + nb * 8 + 2 * quad + c) * N0 + rbase + 8 * i, gw1[nb * 4 + 2 * i + c]);
#pragma unroll
        for (int nb = 0; nb < 2; ++nb)
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int c = 0; c < 2; ++c)      // gW2^T: rows = the N1 input features (M = 64: no half offset)
                    atomicAdd(gW2 + (size_t)(nh * 16 + nb * 8 + 2 * quad + c) * N1 + (rbase - mh * 64) + 8 * i, gw2[nb * 4 + 2 * i + c]);
        // register column sums: shuffle over the 8 row groups of the warp (lanes of equal quad), then shared, then global
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            float v = gb1[k];
#pragma unroll
            for (int off = 4; off <= 16; off <<= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
            if (lane < 4) atomicAdd(&s_colsum[nh * 32 + (k >> 1) * 8 + 2 * quad + (k & 1)], v);
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            float v = gb2[k], g = gwg[k], h = gwh[k];
#pragma unroll
            for (int off = 4; off <= 16; off <<= 1) {
                v += __shfl_xor_sync(0xffffffffu, v, off);
                g += __shfl_xor_sync(0xffffffffu, g, off);
                h += __shfl_xor_sync(0xffffffffu, h, off);
            }
            const int col = nh * 16 + (k >> 1) * 8 + 2 * quad + (k & 1);
            if (lane < 4) {
                atomicAdd(&s_colsum[N1 + col], v);
                atomicAdd(&s_colsum[N1 + N2 + col], g);
                atomicAdd(&s_colsum[N1 + N2 + F + col], h);
            }
        }
        __syncthreads();
        for (int k = tid; k < N1; k += kFusedThreads) if (s_colsum[k] != 0.f) atomicAdd(gb1g + k, s_colsum[k]);
        for (int k = tid; k < N2; k += kFusedThreads) if (s_colsum[N1 + k] != 0.f) atomicAdd(gb2g + k, s_colsum[N1 + k]);
        for (int k = tid; k < 2 * F; k += kFusedThreads) if (s_colsum[N1 + N2 + k] != 0.f) atomicAdd(gwp + k, s_colsum[N1 + N2 + k]);
    }
    // loss and regulariser norms
    {
        const int nv = p.has_reg ? 11 : 1;
#pragma unroll
        for (int k = 0; k < 11; ++k) {
            if (k >= nv) break;
            float v = k == 0 ? acc_loss : (k <= 5 ? acc_l1[k - 1] : acc_s2[k - 6]);
#pragma unroll
            for (int off = 16; off >= 1; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
            if (lane == 0) atomicAdd(&s_red[k], (double)v);
        }
        __syncthreads();
        if (tid < nv && s_red[tid] != 0.0) atomicAdd(p.red + tid, s_red[tid]);
    }
}

template <int F>
static int launch_neumf_fused_f(const FusedParams &p, cudaStream_t st)
{
    using L = FusedLayout<F>;
    // the dynamic shared-memory limit is a per-device function attribute: remember, per calling thread, the devices it was
    // set on (bit d for device d < 64; devices beyond set it on every launch)
    static thread_local unsigned long long attr_set = 0ull;
    int dev = 0;
    DRB_CUDA(cudaGetDevice(&dev));
    const unsigned long long bit = dev < 64 ? 1ull << dev : 0ull;
    if (!(attr_set & bit) || bit == 0ull) {
        DRB_CUDA(cudaFuncSetAttribute(neumf_fused_kernel<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L::BYTES));
        attr_set |= bit;
    }
    long long tiles = (p.B + kFusedTile - 1) / kFusedTile;
    int grid = (int)(tiles < (long long)sm_count() ? tiles : (long long)sm_count());
    if (grid < 1) grid = 1;
    neumf_fused_kernel<F><<<grid, kFusedThreads, L::BYTES, st>>>(p);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}

// The warpgroup split of the epilogues is written for factors = 32 (tower 128 -> 64 -> 32, BASELINE config 3); other shapes
// use the layer-wise path.
static bool neumf_fused_supported(int F, int L, int mode, float dropout)
{
    return L == 2 && mode == 0 && dropout == 0.f && F == 32;
}

static int launch_neumf_fused(int F, const FusedParams &p, cudaStream_t st)
{
    if (F == 32) return launch_neumf_fused_f<32>(p, st);
    DRB_REQUIRE(false, "neumf fused tower: unsupported factors=%d", F);
}

}  // namespace drb
