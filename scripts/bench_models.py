"""Secondary measurements (not the driver's bench): BASELINE configs 3, 4, 5 on one GPU.

    python scripts/bench_models.py lightgcn|neumf|mf-netflix [--batch B] [--steps K]
Prints one JSON line per run: triples/s with CUDA events around K steps after warm-up.
"""
import argparse
import json
import sys

import torch

sys.path.insert(0, ".")
from daisyrec_b200 import ops  # noqa: E402
from daisyrec_b200.utils.synthetic import SHAPES, make_interactions  # noqa: E402


def timed(fn, warm, steps):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def batches(U, I, n, dev, d=None):
    g = torch.Generator(device=dev); g.manual_seed(3)
    if d is not None:                                       # real (u,i) pairs + uniform negatives
        idx = torch.randint(0, d["coo_u"].numel(), (n,), device=dev, generator=g)
        bu, bi = d["coo_u"][idx].contiguous(), d["coo_i"][idx].contiguous()
    else:
        bu = torch.randint(0, U, (n,), device=dev, dtype=torch.int32, generator=g)
        bi = torch.randint(0, I, (n,), device=dev, dtype=torch.int32, generator=g)
    bj = torch.randint(0, I, (n,), device=dev, dtype=torch.int32, generator=g)
    return bu, bi, bj


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("what", choices=["lightgcn", "neumf", "mf-netflix", "mf-fit", "mf-fused"])
    ap.add_argument("--batch", type=int, default=0)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--tower", default="fp32", choices=["fp32", "bf16"])
    a = ap.parse_args()
    dev = torch.device("cuda")
    if a.what == "lightgcn":
        U, I, nnz = SHAPES["amazon-book"]
        F, L = 64, 3
        B = a.batch or 65536
        d = make_interactions(U, I, nnz, device=dev)
        row_ptr, col, val = ops.lgcn_norm_adj(d["coo_u"].cpu().numpy(), d["coo_i"].cpu().numpy(), U, I)
        graph = ops.LgcnGraph(row_ptr, col, val, dev)
        E0 = (torch.randn(U + I, F, device=dev) * 0.05).contiguous()
        ws = ops.LgcnWorkspace(U, I, F, "adam", dev)
        hp = ops.hyper(0.01, 0.0, 0.0, "adam")
        bu, bi, bj = batches(U, I, B * 4, dev, d)
        step = [0]

        def fn():
            ops.lgcn_bpr_train_steps(E0, ws, graph, L, bu, bi, bj, B, step[0] % 4, 1, hp, adam_step0=step[0], check=False)
            step[0] += 1
        ms = timed(fn, 3, a.steps)
        nnzA = int(row_ptr[-1])
        alg = 2 * L * (nnzA * (8 + 4 * F) + (U + I) * 4 * F) + B * (24 * F + 12)
        print(json.dumps(dict(model="LightGCN", shape="amazon-book", U=U, I=I, nnzA=nnzA, F=F, L=L, batch=B, ms_per_step=ms,
                              triples_per_s=B / ms * 1e3, alg_bytes_per_step=alg, alg_GBps=alg / ms / 1e6,
                              spmm_segments=graph.nseg)))
    elif a.what == "neumf":
        U, I, _ = SHAPES["ml-20m"]
        F, L = 32, 2
        B = a.batch or 262144
        D = F * 2 ** (L - 1)
        tabs = [(torch.randn(s, device=dev) * 0.05).contiguous() for s in ((U, F), (I, F), (U, D), (I, D))]
        W = (torch.randn(ops.neumf_param_count(F, L), device=dev) * 0.1).contiguous()
        ws = ops.NeumfWorkspace(U, I, F, L, "adam", 2 * B, dev)
        hp = ops.hyper(0.001, 0.001, 0.001, "adam")
        bu, bi, bj = batches(U, I, B * 4, dev)
        step = [0]

        def fn():
            ops.neumf_bpr_train_steps(tabs, W, ws, bu, bi, bj, B, step[0] % 4, 1, hp, adam_step0=step[0], check=False,
                                      tower_dtype=1 if a.tower == 'bf16' else 0)
            step[0] += 1
        ms = timed(fn, 3, a.steps)
        flop = 0
        n_in = 2 * D
        for _ in range(L):
            flop += 2 * n_in * (n_in // 2)
            n_in //= 2
        flop_triple = 2 * 3 * flop                          # 2 items x (fwd + 2 bwd GEMMs)
        print(json.dumps(dict(model="NeuMF", shape="ml-20m", F=F, L=L, batch=B, ms_per_step=ms, triples_per_s=B / ms * 1e3,
                              tower_TFLOPs=B * flop_triple / ms / 1e9, tower="fp32 CUDA cores" if a.tower == "fp32" else "bf16 wgmma (register accumulators)")))
    elif a.what == "mf-fused":
        # throughput mode: negatives drawn inside the step kernel (Philox + k-th complement over the CSR row)
        U, I, nnz = SHAPES["ml-20m"]
        F, B, K = 64, a.batch or (1 << 20), 16
        d = make_interactions(U, I, nnz, device=dev)
        P = (torch.randn(U, F, device=dev) * 0.01).contiguous(); Q = (torch.randn(I, F, device=dev) * 0.01).contiguous()
        ws = ops.MFWorkspace(U, I, F, "sgd", dev)
        hp = ops.hyper(0.01, 0.001, 0.001)
        g = torch.Generator(device=dev); g.manual_seed(5)
        idx = torch.randint(0, d["coo_u"].numel(), (B * K,), device=dev, generator=g)
        bu, bi = d["coo_u"][idx].contiguous(), d["coo_i"][idx].contiguous()
        bj = torch.randint(0, I, (B * K,), device=dev, dtype=torch.int32, generator=g)
        ms_f = timed(lambda: ops.mf_bpr_train_steps_fused_neg(P, Q, ws, bu, bi, d["row_ptr"], d["col"], 1, B, 0, K, hp, check=False), 1, 3) / K
        ms_t = timed(lambda: ops.mf_bpr_train_steps(P, Q, ws, bu, bi, bj, B, 0, K, hp, check=False), 1, 3) / K
        print(json.dumps(dict(model="MF", shape="ml-20m", F=F, batch=B, fused_sampler_ms_per_step=ms_f,
                              fused_sampler_triples_per_s=B / ms_f * 1e3, table_mode_ms_per_step=ms_t,
                              table_mode_triples_per_s=B / ms_t * 1e3)))
    elif a.what == "mf-fit":
        # wall-clock of the drop-in API at config-2 scale: MF(config).fit(DataLoader over the 80 M sampler triples)
        import logging, time as _t
        sys.path.insert(0, ".")
        import bench as Bn
        from daisyrec_b200.model.MFRecommender import MF
        from daisyrec_b200.utils.dataset import BasicDataset, get_dataloader
        from daisyrec_b200.utils.sampler import TripleArray
        d, triples = Bn.build_workload("ml-20m", dev, 4, 2022, "cuda")
        host = triples.cpu().numpy().view(TripleArray)
        host._drb_device = triples
        for engine in ("torch", "device"):
            cfg = dict(gpu="", logger=logging.getLogger("b"), lr=0.01, reg_1=0.001, reg_2=0.001, epochs=2, topk=50,
                       user_num=d["user_num"], item_num=d["item_num"], factors=64, loss_type="BPR", optimizer="default",
                       init_method="default", early_stop=False, progress=False, shuffle_engine=engine)
            model = MF(cfg)
            loader = get_dataloader(BasicDataset(host), batch_size=a.batch or (1 << 20), shuffle=True)
            torch.cuda.synchronize(); t0 = _t.time()
            model.fit(loader)
            torch.cuda.synchronize(); dt = _t.time() - t0
            print(json.dumps(dict(model="MF.fit drop-in", shuffle_engine=engine, epochs=2, triples=int(host.shape[0]),
                                  wall_s=dt, triples_per_s_wall=2 * host.shape[0] / dt)))
    else:
        U, I, nnz = SHAPES["netflix"]
        F = 128
        B = a.batch or (1 << 20)
        P = (torch.randn(U, F, device=dev) * 0.01).contiguous()
        Q = (torch.randn(I, F, device=dev) * 0.01).contiguous()
        ws = ops.MFWorkspace(U, I, F, "sgd", dev)
        hp = ops.hyper(0.01, 0.001, 0.001)
        K = 16
        bu, bi, bj = batches(U, I, B * K, dev)
        bi = (I * torch.rand(B * K, device=dev).pow(2.0)).to(torch.int32).clamp_(0, I - 1)

        def fn():
            ops.mf_bpr_train_steps(P, Q, ws, bu, bi, bj, B, 0, K, hp, check=False)
        ms = timed(fn, 1, max(1, a.steps // 4)) / K
        print(json.dumps(dict(model="MF", shape="netflix", U=U, I=I, F=F, batch=B, ms_per_step=ms, triples_per_s=B / ms * 1e3,
                              alg_GBps=B * (24 * F + 12) / ms / 1e6)))


if __name__ == "__main__":
    main()
