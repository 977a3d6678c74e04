"""Where the time of one BPR-MF step goes, at the bench's workload (ML-20M shape, F = 64, SGD, batch 1 048 576).

Prints one JSON line per measurement (ms per step, CUDA events around launches that end in a synchronise):
  fused         ops.mf_bpr_train_steps: the persistent launch bench.py times
  phase1        drb_mf_bpr_phase(phase=1), one launch per step: gathers, dots, loss, norms and the gradient REDs
  phase2        drb_mf_bpr_phase(phase=2), one launch per step, each after a phase-1 launch: the dense sweep
  loss_only     ops.mf_bpr_loss: phase 1 without any RED (loads and loss only), one launch per step
  fused_sorted  the fused launch on planes sorted by user within each step (same batches, other fp32 summation order)
and a first line with the card, its power limit and SM clocks.  Usage: python scripts/probe_mf_phases.py [steps] [reps]
"""
import ctypes as C
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from daisyrec_b200 import _lib as L  # noqa: E402
from daisyrec_b200 import ops  # noqa: E402
from daisyrec_b200.utils.synthetic import init_tables  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        out = repr(e)
    return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))


def timed(fn, steps, reps):
    """best of `reps` windows of `steps` steps (fn(s) runs step s), ms per step"""
    best = None
    for _ in range(reps):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for s in range(steps):
            fn(s)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / steps
        best = ms if best is None else min(best, ms)
    return best


def main():
    K = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    seed, B, F = 2022, 1 << 20, 64
    d, triples = bench.build_workload("ml-20m", dev, 4, seed, "cuda")
    U, I = d["user_num"], d["item_num"]
    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    perm = torch.randperm(triples.shape[0], generator=g, device=dev)
    bu, bi, bj = ops.gather_triples(triples, perm)
    del perm, triples
    bu, bi, bj = bu[:K * B].contiguous(), bi[:K * B].contiguous(), bj[:K * B].contiguous()
    # the same batches, each sorted by user (outside any timed region)
    su, order = torch.sort(bu.view(K, B).long(), dim=1, stable=True)
    su = su.to(torch.int32).reshape(-1).contiguous()
    si = torch.gather(bi.view(K, B), 1, order).reshape(-1).contiguous()
    sj = torch.gather(bj.view(K, B), 1, order).reshape(-1).contiguous()
    del order
    hp = ops.hyper(**bench.HYPER)
    print(json.dumps({"card": card(), "U": U, "I": I, "F": F, "batch": B, "steps": K, "reps": reps,
                      "step_variant": ops.mf_step_variant(F, U + I), "selfcheck_ms": ops.mf_step_selfcheck_ms(F, U + I)}),
          flush=True)
    P0, Q0 = init_tables(U, I, F, seed, dev)

    def fresh():
        return P0.clone(), Q0.clone(), ops.MFWorkspace(U, I, F, "sgd", dev)

    def report(name, ms):
        print(json.dumps({"what": name, "ms_per_step": ms, "G_triples_per_s": B / ms / 1e6}), flush=True)

    for name, planes in (("fused", (bu, bi, bj)), ("fused_sorted", (su, si, sj))):
        P, Q, ws = fresh()
        ops.mf_bpr_train_steps(P, Q, ws, *planes, B, 0, 2, hp, check=False)            # warm-up
        report(name, timed(lambda s: ops.mf_bpr_train_steps(P, Q, ws, *planes, B, 0, K, hp, check=False), 1, reps) / K)

    P, Q, ws = fresh()
    loss = torch.empty(1, dtype=torch.float64, device=dev)

    def phase(ph, s):
        L.check(L.lib().drb_mf_bpr_phase(P.data_ptr(), Q.data_ptr(), ws.buf.data_ptr(), U, I, F, bu.data_ptr(), bi.data_ptr(),
                                         bj.data_ptr(), s * B, B, ph, C.byref(hp), 0, loss.data_ptr(),
                                         C.c_void_p(torch.cuda.current_stream().cuda_stream)))

    for s in range(2):                                                                   # warm-up
        phase(1, s); phase(2, s)
    t1, t2 = [], []
    for _ in range(reps):
        evs = []
        torch.cuda.synchronize()
        for s in range(K):
            e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            e[0].record(); phase(1, s); e[1].record(); phase(2, s); e[2].record()
            evs.append(e)
        torch.cuda.synchronize()
        t1.append(sum(e[0].elapsed_time(e[1]) for e in evs) / K)
        t2.append(sum(e[1].elapsed_time(e[2]) for e in evs) / K)
    report("phase1", min(t1))
    report("phase2", min(t2))

    P, Q, ws = fresh()
    ops.mf_bpr_loss(P, Q, ws, bu[:B], bi[:B], bj[:B], hp)
    report("loss_only", timed(lambda s: ops.mf_bpr_loss(P, Q, ws, bu[s * B:(s + 1) * B], bi[s * B:(s + 1) * B],
                                                         bj[s * B:(s + 1) * B], hp), K, reps))


if __name__ == "__main__":
    main()
