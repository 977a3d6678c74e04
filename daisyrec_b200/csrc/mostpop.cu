// mostpop.cu -- MostPop (daisy/model/PopRecommender.py, Ji et al. 2020) on the device.
//
//   drb_mostpop_fit     value_counts of the item column (every row, duplicates included) by 64-bit integer atomics, so the
//                       counts do not depend on the order the rows are added in, then item_score = cnt / (1 + cnt) in fp64,
//                       one correctly rounded division as numpy's.  Ids outside [0, item_num) are counted, not added.
//   drb_mostpop_gather  scores[r][c] = item_score[cands[r][c]], the candidate scores drb_itemknn_topk ranks.
#include "common.cuh"

namespace drb {

__global__ void mostpop_count_kernel(const int64_t *__restrict__ ids, long long n, int I, unsigned long long *__restrict__ cnt,
                                     unsigned long long *__restrict__ bad)
{
    unsigned long long mine = 0;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
        const long long i = ids[k];
        if (i < 0 || i >= I) ++mine;
        else atomicAdd(cnt + i, 1ull);
    }
    if (mine) atomicAdd(bad, mine);
}

__global__ void mostpop_score_kernel(const unsigned long long *__restrict__ cnt, int I, double *__restrict__ cnt_f,
                                     double *__restrict__ score)
{
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < I; i += gridDim.x * blockDim.x) {
        const double c = (double)cnt[i];
        cnt_f[i] = c;
        score[i] = __ddiv_rn(c, __dadd_rn(1.0, c));
    }
}

__global__ void mostpop_gather_kernel(const double *__restrict__ score, const int64_t *__restrict__ cands, long long total,
                                      double *__restrict__ out)
{
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < total; k += (long long)gridDim.x * blockDim.x)
        out[k] = score[cands[k]];
}

}  // namespace drb

using namespace drb;

extern "C" size_t drb_mostpop_workspace_bytes(int32_t item_num)
{
    return item_num > 0 ? sizeof(unsigned long long) * ((size_t)item_num + 1) : 0;
}

extern "C" int drb_mostpop_fit(const int64_t *d_ids, int64_t n, int32_t item_num, void *d_ws, double *d_cnt, double *d_score,
                               int64_t *h_bad, void *stream)
{
    DRB_REQUIRE(d_ws && d_cnt && d_score && h_bad && item_num > 0 && n >= 0 && (n == 0 || d_ids), "mostpop_fit: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    unsigned long long *cnt = (unsigned long long *)d_ws, *bad = cnt + item_num;
    DRB_CUDA(cudaMemsetAsync(d_ws, 0, drb_mostpop_workspace_bytes(item_num), st));
    if (n > 0) mostpop_count_kernel<<<grid_for(n, 256), 256, 0, st>>>(d_ids, n, item_num, cnt, bad);
    mostpop_score_kernel<<<grid_for(item_num, 256), 256, 0, st>>>(cnt, item_num, d_cnt, d_score);
    DRB_CUDA(cudaGetLastError());
    unsigned long long h = 0;
    DRB_CUDA(cudaMemcpyAsync(&h, bad, sizeof(h), cudaMemcpyDeviceToHost, st));
    DRB_CUDA(cudaStreamSynchronize(st));
    *h_bad = (int64_t)h;
    return DRB_OK;
}

extern "C" int drb_mostpop_gather(const double *d_score, const int64_t *d_cands, int64_t total, double *d_out, void *stream)
{
    DRB_REQUIRE(d_score && d_cands && d_out && total >= 0, "mostpop_gather: bad arguments");
    if (total == 0) return DRB_OK;
    mostpop_gather_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(d_score, d_cands, total, d_out);
    DRB_CUDA(cudaGetLastError());
    return DRB_OK;
}
