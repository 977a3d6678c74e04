"""Where the time of one BPR-MF step goes, at the bench's workload (ML-20M shape, F = 64, SGD, batch 1 048 576).

Prints one JSON line per measurement (ms per step, CUDA events around launches that end in a synchronise):
  fused         ops.mf_bpr_train_steps: the persistent launch bench.py times
  phase1        drb_mf_bpr_phase(phase=1), one launch per step: gathers, dots, loss, norms and the gradient REDs
  phase2        drb_mf_bpr_phase(phase=2), one launch per step, each after a phase-1 launch: the dense sweep
  loss_only     ops.mf_bpr_loss: phase 1 without any RED (loads and loss only), one launch per step
  fused_sorted  the fused launch on planes sorted by user within each step (same batches, other fp32 summation order)
and a first line with the card, its power limit and SM clocks.  Usage: python scripts/probe_mf_phases.py [steps] [reps]

With --timers it instead builds the step library once more with -DDRB_PHASE_TIMERS (as scripts/build_variants.sh builds its
A/B variants: mf_bpr.cu alone, linked with the other objects of the library build, into daisyrec_b200/lib/variants/), runs one
fused launch of `steps` steps on it, and prints per section of the staged user-bucketed step the median over steps of the
maximum over CTAs (ms), and of the time between the last CTAs to reach its two boundaries (the critical path).
"""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

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


# boundaries written by phase_mark (step_kernel.cuh), per step: 0 step start, 1 histogram done, 2 after its barrier, 3 scan and
# reservation done, 4 scatter done, 5 after its barrier and the count zeroing, 6 phase 1 done, 7 after its barrier, 8 item sweep
# done; launch start (9), norm-cache fill done (10) and after its barrier (11) in step 0's slots
SECTIONS = (("histogram", 0, 1), ("barrier_hist", 1, 2), ("scan_reserve", 2, 3), ("scatter", 3, 4), ("barrier_scatter", 4, 5),
            ("phase1", 5, 6), ("barrier_phase1", 6, 7), ("item_sweep", 7, 8), ("barrier_step", 8, None))


def timer_lib():
    """the probe build of the library (rebuilt when mf_bpr.cu or a header is newer)"""
    from daisyrec_b200 import _build
    out = os.path.join(_build.LIBDIR, "variants")
    so = os.path.join(out, "lib_phase_timers.so")
    if not _build._stale(so, [os.path.join(_build.CSRC, f) for f in os.listdir(_build.CSRC)]):
        return so
    _build.build()
    os.makedirs(out, exist_ok=True)
    obj = os.path.join(out, "mf_bpr_phase_timers.o")
    subprocess.check_call([_build.nvcc()] + _build.ARCH + _build.FLAGS + ["-DDRB_PHASE_TIMERS", "-c",
                          os.path.join(_build.CSRC, "mf_bpr.cu"), "-o", obj])
    others = [os.path.join(_build.LIBDIR, f.replace(".cu", ".o")) for f in _build.SOURCES if f != "mf_bpr.cu"]
    subprocess.check_call([_build.nvcc()] + _build.ARCH + ["-shared", "-cudart", "static", "-o", so, obj] + others + ["-ldl"])
    os.remove(obj)
    return so


def phase_timers(K):
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
    hp = ops.hyper(**bench.HYPER)
    P, Q = init_tables(U, I, F, seed, dev)
    ws = ops.MFWorkspace(U, I, F, "sgd", dev)
    ops.mf_bpr_train_steps(P, Q, ws, bu, bi, bj, B, 0, 2, hp, check=False)            # warm-up
    ops.mf_bpr_train_steps(P, Q, ws, bu, bi, bj, B, 0, K, hp, check=False)
    torch.cuda.synchronize()
    lib = L.lib()
    assert lib.drb_mf_last_step_mode() == 2 and lib.drb_mf_last_step_staged() == 1, "the launch did not run the staged form"
    dims = (C.c_int32 * 3)()
    buf = np.zeros(96 * 12 * 512 + 1, np.uint64)
    lib.drb_phase_timers.restype = C.c_int
    L.check(lib.drb_phase_timers(C.c_void_p(buf.ctypes.data), dims))
    ns, nm, nc = dims[0], dims[1], dims[2]
    assert ns * nm * nc <= buf.size
    t = buf[:ns * nm * nc].reshape(ns, nm, nc).astype(np.int64)
    ctas = int((t[0, 0] != 0).sum())
    steps = min(K, ns)
    t = t[:steps, :, :ctas]
    print(json.dumps({"card": card(), "U": U, "I": I, "F": F, "batch": B, "steps": steps, "ctas": ctas}), flush=True)
    res = {}
    step_ms = np.median(np.diff(t[:, 0, :].max(axis=1))) / 1e6
    for name, a, b in SECTIONS:
        n = steps - 1 if b is None else steps
        end = t[1:n + 1, 0] if b is None else t[:n, b]
        per_cta = (end - t[:n, a]).max(axis=1)
        crit = end.max(axis=1) - t[:n, a].max(axis=1)
        res[name] = {"max_cta_ms": float(np.median(per_cta)) / 1e6, "critical_ms": float(np.median(crit)) / 1e6}
    fill = {"norm_fill_ms": float((t[0, 10] - t[0, 9]).max()) / 1e6, "barrier_fill_ms": float((t[0, 11] - t[0, 10]).max()) / 1e6}
    print(json.dumps({"what": "phase_timers", "step_ms": float(step_ms), "sections": res, "launch": fill}), flush=True)
    for name, _, _ in SECTIONS:
        print(f"  {name:16s} max over CTAs {res[name]['max_cta_ms']:.4f} ms   critical path {res[name]['critical_ms']:.4f} ms",
              flush=True)


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
    if "--timers" in sys.argv:
        sys.argv.remove("--timers")
        os.environ["DRB_LIB_PATH"] = timer_lib()
        phase_timers(int(sys.argv[1]) if len(sys.argv) > 1 else 40)
    else:
        main()
