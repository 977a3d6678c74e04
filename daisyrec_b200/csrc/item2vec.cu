// item2vec.cu -- the Item2Vec training step and user-embedding build.
//
// Stands behind Item2Vec.fit / calc_loss (daisy/model/Item2VecRecommender.py:16-107): BCEWithLogitsLoss(sum) of
// shared[t] . shared[c] against the label, no regulariser, autograd summing both operands' contributions into the one shared
// table, then optim.SGD / Adam.  The step is the point-wise CL branch of the GEN step kernel (step_kernel.cuh) switched to
// one tied table (StepParams::U = 0): both rows gather from Q, both gradients land in gQ (t == c adds 2 g e_t), and phase 2
// sweeps the item table alone.  After fit, user_embedding[u] = sum of shared[i] over the user's train items: a segmented row
// sum over the user -> item CSR, one warp per user.
#include "step.cuh"

namespace drb {

__global__ void i2v_user_sum_kernel(const float *__restrict__ Q, int F, const int64_t *__restrict__ row_ptr,
                                    const int32_t *__restrict__ col, int U, float *__restrict__ P)
{
    const int lane = threadIdx.x & 31;
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long u = warp; u < U; u += nwarps) {
        const long long b = row_ptr[u], e = row_ptr[u + 1];
        if (b == e) continue;   // not in train_ur: the row keeps its initial values
        for (int f0 = 0; f0 < F; f0 += 32) {
            const int f = f0 + lane;
            float s = 0.f;
            for (long long k = b; k < e; ++k)
                if (f < F) s += __ldg(Q + (size_t)__ldg(col + k) * F + f);
            if (f < F) P[(size_t)u * F + f] = s;
        }
    }
}

}  // namespace drb

using namespace drb;

extern "C" size_t drb_i2v_workspace_bytes(int32_t I, int32_t F, int32_t opt)
{
    return carve(nullptr, 0, I, F, opt, nullptr);
}

extern "C" int drb_i2v_workspace_init(void *d_ws, int32_t I, int32_t F, int32_t opt, void *stream)
{
    DRB_REQUIRE(d_ws != nullptr && I > 0 && F > 0, "i2v_workspace_init: bad arguments");
    DRB_CUDA(cudaMemsetAsync(d_ws, 0, carve(nullptr, 0, I, F, opt, nullptr), (cudaStream_t)stream));
    return DRB_OK;
}

extern "C" int drb_i2v_train_steps(float *d_Q, void *d_ws, int32_t I, int32_t F, const int32_t *d_bt, const int32_t *d_bc,
                                   const int32_t *d_blabel, int64_t n, int64_t batch, int64_t first_step, int64_t n_steps,
                                   const drb_hyper *hyper, int64_t adam_step0, int32_t apply, double *d_step_loss,
                                   int32_t sync_and_check, int64_t *nan_step, void *stream)
{
    DRB_REQUIRE(d_Q && d_ws && d_bt && d_bc && d_blabel && hyper && d_step_loss, "i2v_train_steps: null pointer argument");
    DRB_REQUIRE(I > 0 && F > 0 && batch > 0 && n >= 0 && first_step >= 0 && n_steps >= 0, "i2v_train_steps: bad sizes");
    DRB_REQUIRE(hyper->loss == DRB_LOSS_CL, "i2v_train_steps: the skip-gram step is point-wise CL");
    DRB_REQUIRE(hyper->opt == DRB_OPT_SGD || hyper->opt == DRB_OPT_ADAM, "i2v_train_steps: optimizer id %d (SGD or Adam)",
                hyper->opt);
    DRB_REQUIRE(hyper->reg_1 == 0.f && hyper->reg_2 == 0.f, "i2v_train_steps: Item2Vec has no regulariser");
    DRB_REQUIRE((first_step + n_steps - 1) * batch < n || n_steps == 0 || n == 0, "steps [%lld,%lld) exceed %lld rows",
                (long long)first_step, (long long)(first_step + n_steps), (long long)n);
    DRB_REQUIRE(apply || n_steps == 1, "i2v_train_steps: apply=0 evaluates the loss of ONE batch");
    if (n_steps == 0) return DRB_OK;
    StepParams p = one_step(hyper, 0, I, F, d_bt, d_bc, d_blabel, batch, adam_step0);
    p.n = n; p.first_step = first_step; p.n_steps = n_steps;
    p.P = d_Q; p.Q = d_Q;
    carve(d_ws, 0, I, F, hyper->opt, &p.ws);
    p.ws.gP = p.ws.gQ;
    p.dense_hint = 1;   // the claim mode's per-triple row claims assume two tables
    p.step_loss = d_step_loss;
    p.apply = apply;
    cudaStream_t st = (cudaStream_t)stream;
    int rc = launch_steps(p, st);
    if (rc != DRB_OK) return rc;
    if (sync_and_check) return check_nan(d_ws, st, nan_step);
    return DRB_OK;
}

extern "C" int drb_i2v_user_embedding(const float *d_Q, int32_t F, const int64_t *d_row_ptr, const int32_t *d_col, int32_t U,
                                      float *d_P, void *stream)
{
    DRB_REQUIRE(d_Q && d_row_ptr && d_P && F > 0 && U > 0, "i2v_user_embedding: bad arguments");
    i2v_user_sum_kernel<<<grid_for((long long)U * 32, 256), 256, 0, (cudaStream_t)stream>>>(d_Q, F, d_row_ptr, d_col, U, d_P);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}
