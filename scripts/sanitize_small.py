"""Tiny run of every kernel family, meant for `compute-sanitizer --tool memcheck|racecheck python scripts/sanitize_small.py`."""
import sys
import numpy as np
import torch
sys.path.insert(0, ".")
from daisyrec_b200 import ops

rng = np.random.default_rng(0)
dev = "cuda"
U, I, F, B, G = 300, 200, 64, 1000, 4
t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
# sampler
nnz = 4000
cu = rng.integers(U, size=nnz).astype(np.int32); ci = rng.integers(I, size=nnz).astype(np.int32)
key = np.unique(cu.astype(np.int64) * (1 << 32) + ci)
row_ptr = np.zeros(U + 1, np.int64); np.add.at(row_ptr, (key >> 32) + 1, 1); row_ptr = np.cumsum(row_ptr)
col = (key & 0xFFFFFFFF).astype(np.int32)
draws = ops.sampler_draw_mt19937(ops.mt19937_seed(1), row_ptr, U, I, G)
js = ops.sampler_kth_complement(t(row_ptr), t(col), t(draws), I)
tr = ops.sampler_explode(t(cu), t(ci), js)
d2, bad = ops.sampler_draw_philox(3, 0, t(row_ptr), U, I, G)
bu, bi, bj = ops.gather_triples(tr, torch.randperm(tr.shape[0], device=dev))
# MF: fused steps (dense + claim modes), Adam, loss only, host paths
P = t((rng.standard_normal((U, F)) * .1).astype(np.float32)); Q = t((rng.standard_normal((I, F)) * .1).astype(np.float32))
for opt in ("sgd", "adam"):
    ws = ops.MFWorkspace(U, I, F, opt, dev)
    hp = ops.hyper(0.01, 0.001, 0.001, opt)
    ops.mf_bpr_train_steps(P, Q, ws, bu, bi, bj, B, 0, 5, hp)
    ops.mf_bpr_train_steps(P, Q, ws, bu, bi, bj, 37, 0, 9, hp)            # claim mode, unaligned tiles
    ops.mf_bpr_loss(P, Q, ws, bu[:B], bi[:B], bj[:B], hp)
hb = [x[:3 * B].cpu().pin_memory() for x in (bu, bi, bj)]
ws = ops.MFWorkspace(U, I, F, "sgd", dev); hp = ops.hyper(0.01, 0.001, 0.001)
ops.mf_bpr_train_steps_host(P, Q, ws, *hb, B, 3, hp)
ops.mf_bpr_train_step_host(P, Q, ws, *[x[:B] for x in hb], hp, ops.stage_buffer(B, dev))
# rank
users = t(rng.integers(U, size=9).astype(np.int64)); cands = t(rng.integers(I, size=(9, 150)).astype(np.int64))
ops.mf_rank(P, Q, users, cands, 20); ops.mf_full_rank(P, Q, users, 20)
ops.mf_predict(P, Q, users.to(torch.int32), cands[:, 0].to(torch.int32).contiguous())
# LightGCN
rp, cc, vv = ops.lgcn_norm_adj(cu, ci, U, I)
graph = ops.LgcnGraph(rp, cc, vv, dev)
E0 = t((rng.standard_normal((U + I, F)) * .1).astype(np.float32))
lws = ops.LgcnWorkspace(U, I, F, "adam", dev)
ops.lgcn_propagate(E0, lws, graph, 2)
ops.lgcn_bpr_train_steps(E0, lws, graph, 2, bu, bi, bj, B, 0, 2, ops.hyper(0.01, 0.001, 0.001, "adam"))
# NeuMF fp32 + bf16 (wgmma) + dropout
Fn, L = 32, 2; D = Fn * 2
tabs = [t((rng.standard_normal(s) * .2).astype(np.float32)) for s in ((U, Fn), (I, Fn), (U, D), (I, D))]
W = t((rng.standard_normal(ops.neumf_param_count(Fn, L)) * .1).astype(np.float32))
nws = ops.NeumfWorkspace(U, I, Fn, L, "adam", 2 * B, dev)
for dt in (0, 1):
    ops.neumf_bpr_train_steps(tabs, W, nws, bu, bi, bj, B, 0, 2, ops.hyper(0.001, 0.001, 0.001, "adam"), tower_dtype=dt,
                              dropout=0.3, dropout_seed=7)
    sc = ops.neumf_scores(tabs, W, nws, users, cands, 150, tower_dtype=dt)
    ops.topk_from_scores(sc, cands, 10)
torch.cuda.synchronize()
print("sanitize_small: all kernels ran")
