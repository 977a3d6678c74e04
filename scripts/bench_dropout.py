"""NGCF and NFM step times under each dropout setting, at bench.py's f_ngcf and f_nfm shapes.

NGCF: Amazon-Book shape (utils.synthetic SHAPES, adjacency built on the device), widths 64/64/64/64, Adam, B = 65 536 --
      dropout 0; mess_dropout 0.1 with 'torch' (host masks) and 'philox'; mess 0.1 + node_dropout 0.1 with 'philox'.
NFM:  ML-20M shape, F = 64, one hidden layer, BatchNorm, relu, Adam, B = 262 144 -- dropout 0; 0.5 'torch'; 0.5 'philox'.

The 'torch' rows time what the model classes do with dropout_engine 'torch': per step the masks are drawn with bernoulli_ on
torch's CPU generator and uploaded, then the step runs; they are host-bound and timed over a few steps only.  The device rows
are timed over --steps steps after --warmup, in --rounds alternating rounds; the median round is reported.  Prints one JSON
line per setting, with the card's name and power limit read in the same run.

    python scripts/bench_dropout.py [--steps 20 --warmup 3 --rounds 3 --host-steps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def timed_ms(step, warmup, steps):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(steps):
        step()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) / steps * 1e3


def ngcf_settings(dev):
    from daisyrec_b200 import ops
    from daisyrec_b200.utils.synthetic import SHAPES, make_interactions
    U, I, nnz = SHAPES["amazon-book"]
    g = torch.Generator(device=dev); g.manual_seed(12)
    da = make_interactions(U, I, nnz, seed=0, device=dev)
    graph = ops.LgcnGraph(*ops.lgcn_build_adj(da["coo_u"], da["coo_i"], U, I), dev)
    dims = [64, 64, 64, 64]
    E0 = (torch.randn(U + I, dims[0], device=dev, generator=g) * 0.05).contiguous()
    W = (torch.randn(ops.ngcf_param_count(dims), device=dev, generator=g) * 0.1).contiguous()
    ws = ops.NgcfWorkspace(U, I, dims, "adam", dev)
    B = 65536
    idx = torch.randint(0, da["coo_u"].numel(), (4 * B,), device=dev, generator=g)
    bu, bi = da["coo_u"][idx].contiguous(), da["coo_i"][idx].contiguous()
    bj = torch.randint(0, I, (4 * B,), device=dev, dtype=torch.int32, generator=g)
    hp = ops.hyper(0.001, 0.0, 0.001, "adam")
    graph.edge_mirror()                                   # built once per graph, outside the timed steps
    k = [0]
    n = U + I

    def run(engine, mess, node):
        def step():
            s = k[0] % 4
            if engine == "philox":
                ops.ngcf_bpr_train_steps_philox(E0, W, ws, graph, bu, bi, bj, B, s, 1, hp, adam_step0=k[0], check=False, seed=7,
                                                forward0=k[0], mess_dropout=mess, node_dropout=node)
            elif mess > 0:
                keep = torch.cat([torch.empty(n, w).bernoulli_(1 - mess).to(torch.uint8).reshape(-1) for w in dims[1:]]).to(dev)
                ops.ngcf_bpr_train_steps(E0, W, ws, graph, bu, bi, bj, B, s, 1, hp, adam_step0=k[0], check=False, dropout=mess,
                                         keep=keep)
            else:
                ops.ngcf_bpr_train_steps(E0, W, ws, graph, bu, bi, bj, B, s, 1, hp, adam_step0=k[0], check=False)
            k[0] += 1
        return step
    desc = f"NGCF+BPR amazon-book shape ({U}x{I}, adjacency nnz={int(graph.col.numel())}), widths {dims}, Adam, B={B}"
    return desc, B, [("dropout 0", run("none", 0.0, 0.0), False),
                     ("mess 0.1 'torch'", run("torch", 0.1, 0.0), True),
                     ("mess 0.1 'philox'", run("philox", 0.1, 0.0), False),
                     ("mess 0.1 + node 0.1 'philox'", run("philox", 0.1, 0.1), False)]


def nfm_settings(dev):
    from daisyrec_b200 import ops
    from daisyrec_b200.utils.synthetic import SHAPES, init_tables
    U, I, _ = SHAPES["ml-20m"]
    F, Ln, bn, B = 64, 1, True, 1 << 18
    g = torch.Generator(device=dev); g.manual_seed(11)
    P, Q = init_tables(U, I, F, 4, dev)
    P.mul_(10.0); Q.mul_(10.0)
    bias = torch.zeros(U + I + 1, dtype=torch.float32, device=dev)
    N = (torch.randn(ops.nfm_param_count(F, Ln, bn), device=dev, generator=g) * 0.1).contiguous()
    N[0:F] = 1.0
    o = 2 * F + F * F + F
    N[o:o + F] = 1.0
    R = torch.zeros(2 * 2 * F, dtype=torch.float32, device=dev)
    R[F:2 * F] = 1.0; R[3 * F:4 * F] = 1.0
    ws = ops.NfmWorkspace(U, I, F, Ln, bn, "adam", 2 * B, dev)
    hp = ops.hyper(0.001, 0.0, 0.001, "adam")
    nst = 8
    bu = torch.randint(0, U, (nst * B,), device=dev, dtype=torch.int32, generator=g)
    bi = torch.randint(0, I, (nst * B,), device=dev, dtype=torch.int32, generator=g)
    bj = torch.randint(0, I, (nst * B,), device=dev, dtype=torch.int32, generator=g)
    act, k = ops.NFM_ACT["relu"], [0]
    args = (P, Q, bias, N, R, ws, act, bu, bi, bj, B)

    def run(engine, p):
        def step():
            s = k[0] % nst
            if engine == "philox":
                ops.nfm_bpr_train_steps_philox(*args, s, 1, hp, adam_step0=k[0], check=False, dropout=p, seed=7)
            elif p > 0:
                keep = torch.empty(2 * (1 + Ln) * B * F).bernoulli_(1 - p).to(torch.uint8).to(dev)
                ops.nfm_bpr_train_steps(*args, s, 1, hp, adam_step0=k[0], check=False, dropout=p, keep=keep)
            else:
                ops.nfm_bpr_train_steps(*args, s, 1, hp, adam_step0=k[0], check=False)
            k[0] += 1
        return step
    desc = f"NFM+BPR ml-20m shape ({U}x{I}), factors={F}, num_layers={Ln}, batch_norm, relu, Adam, B={B}"
    return desc, B, [("dropout 0", run("none", 0.0), False),
                     ("dropout 0.5 'torch'", run("torch", 0.5), True),
                     ("dropout 0.5 'philox'", run("philox", 0.5), False)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--host-steps", type=int, default=3)
    args = ap.parse_args()
    from daisyrec_b200 import ops
    ops.require_cuda()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    gpu = card()
    for model, build in (("ngcf", ngcf_settings), ("nfm", nfm_settings)):
        desc, B, settings = build(dev)
        times = {name: [] for name, _, _ in settings}
        for _ in range(args.rounds):                    # device settings alternate within each round
            for name, step, host in settings:
                if not host:
                    times[name].append(timed_ms(step, args.warmup, args.steps))
        for name, step, host in settings:
            if host:
                times[name].append(timed_ms(step, 1, args.host_steps))
        base = sorted(times["dropout 0"])[len(times["dropout 0"]) // 2]
        for name, _, host in settings:
            ms = sorted(times[name])[len(times[name]) // 2]
            print(json.dumps({"model": model, "workload": desc, "setting": name, "ms_per_step": round(ms, 3),
                              "triples_per_s": round(B / ms * 1e3), "vs_dropout0": round(ms / base, 3),
                              "rounds_ms": [round(t, 3) for t in times[name]], "host_masks": host, "gpu": gpu}), flush=True)
        del settings
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
