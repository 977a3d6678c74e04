"""PureSVD fit and scoring on one GPU at factors 150 (l = 160); prints a phase table and one JSON line.

Workloads (synthetic.make_interactions, seed 2022, binary values):
* ml20m       the ML-20M shape (U = 138 493, I = 26 744, 20 M rows): U >= I, A = X, n_iter 7;
* netflix     the Netflix shape (U = 480 189, I = 17 770, 100 M rows): A = X, n_iter 7;
* transposed  the ML-20M shape with users and items swapped (U = 26 744 < I = 138 493): A = X^T, n_iter 7;
* i8000       U = 40 000, I = 8 000, 2 M rows, beside the reference's PureSVD.fit from oracle/_ref on the host cores.

Per workload one fit after a warm-up fit of the same shape, timed by phase with CUDA events: the host Omega draw (host clock),
the CSR build, every SpMM (total, per call, and the algorithmic bytes of a call: nnz * l * 8 of gathered panel rows plus the
rows * l * 8 output, beside nnz * 12 of CSR reads), orth, small_svd and factors.  Then rank() for 4 096 users x 1 000 candidates
and full_rank() per user (64 users in one call).

    python scripts/bench_puresvd.py [--workloads ml20m,netflix,transposed,i8000] [--no-reference]
"""
import argparse
import json
import logging
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from daisyrec_b200 import ops  # noqa: E402
from daisyrec_b200.utils import synthetic  # noqa: E402

FACTORS = 150


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in q.split(",")]
        return dict(name=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:  # noqa: BLE001
        return dict(name=torch.cuda.get_device_name(), power_limit=f"not read ({e!r})")


class Marks:
    """CUDA events at phase boundaries: mark(phase) closes the interval since the previous mark under that phase's name."""

    def __init__(self):
        self.events = []
        self.start()

    def start(self):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        self.events.append((None, e))

    def __call__(self, phase):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        self.events.append((phase, e))

    def totals(self):
        torch.cuda.synchronize()
        out, calls = {}, {}
        for (_, a), (phase, b) in zip(self.events, self.events[1:]):
            out[phase] = out.get(phase, 0.0) + a.elapsed_time(b) / 1e3
            calls[phase] = calls.get(phase, 0) + 1
        return out, calls


def fit_phases(d_u, d_i, d_v, U, I, k=FACTORS):
    n, l = min(U, I), k + 10
    transposed, n_iter = U < I, (7 if k < 0.1 * n else 4)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    omega = np.random.RandomState(2019).normal(size=(n, l))
    t_omega = time.perf_counter() - t0
    marks = Marks()
    X = ops.puresvd_csr(d_u, d_i, d_v, U, I)
    marks("csr")
    P, Q, s = ops.puresvd_fit(X, omega, k, n_iter, transposed, mark=marks)
    tot, calls = marks.totals()
    nnz = X.col.numel()
    # per SpMM: nnz gathered panel rows of l doubles, plus the output rows (A Z: rows of A; A^T Z: rows of A^T)
    m = I if transposed else U
    bytes_pair = nnz * l * 8 * 2 + (m + n) * l * 8
    spmm_bytes = bytes_pair * calls["spmm"] / 2
    r = dict(users=U, items=I, rows=nnz, l=l, n_iter=n_iter, transposed=transposed, omega_host_s=t_omega,
             csr_s=tot["csr"], upload_s=tot["upload"], spmm_s=tot["spmm"], spmm_calls=calls["spmm"],
             spmm_ms_per_call=1e3 * tot["spmm"] / calls["spmm"], spmm_bytes_per_call=spmm_bytes / calls["spmm"],
             spmm_csr_bytes_per_call=nnz * 12, spmm_tb_per_s=spmm_bytes / tot["spmm"] / 1e12,
             orth_s=tot["orth"], orth_calls=calls["orth"], small_svd_s=tot["small_svd"], factors_s=tot["factors"])
    r["fit_s"] = t_omega + sum(tot.values())
    return X, P, Q, r


def scoring(P, Q, U, I, n_users=4096, n_cands=1000, n_full=64):
    g = torch.Generator(device="cuda")
    g.manual_seed(0)
    users = torch.randint(U, (n_users,), generator=g, device="cuda")
    cands = torch.randint(I, (n_users, n_cands), generator=g, device="cuda")
    ops.puresvd_rank(P, Q, users, cands, 50)                    # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ops.puresvd_rank(P, Q, users, cands, 50)
    torch.cuda.synchronize()
    t_rank = time.perf_counter() - t0
    fu = users[:n_full].contiguous()
    ops.puresvd_full_rank(P, Q, fu, 50)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ops.puresvd_full_rank(P, Q, fu, 50)
    torch.cuda.synchronize()
    t_full = time.perf_counter() - t0
    return dict(rank_s=t_rank, rank_users_per_s=n_users / t_rank, full_rank_ms_per_user=1e3 * t_full / n_full)


def workload(U, I, nnz):
    if U < I:                                                   # the transposed shape: the ML-20M rows with the roles swapped
        d = synthetic.make_interactions(I, U, nnz, device="cuda")
        d_u, d_i = d["coo_i"], d["coo_u"]
    else:
        d = synthetic.make_interactions(U, I, nnz, device="cuda")
        d_u, d_i = d["coo_u"], d["coo_i"]
    d_v = torch.ones(d_u.numel(), dtype=torch.float64, device="cuda")
    fit_phases(d_u, d_i, d_v, U, I)                             # warm-up fit of the same shape
    torch.cuda.empty_cache()
    X, P, Q, r = fit_phases(d_u, d_i, d_v, U, I)
    r.update(scoring(P, Q, U, I))
    del X, P, Q, d
    torch.cuda.empty_cache()
    return r


def reference_arm(U=40000, I=8000, nnz=2_000_000):
    """The reference's PureSVD.fit (sklearn on the host) and the GPU fit on the same rows."""
    import pandas as pd
    d = synthetic.make_interactions(U, I, nnz, device="cpu")
    u, i = d["coo_u"].numpy(), d["coo_i"].numpy()
    args = (torch.from_numpy(u).cuda(), torch.from_numpy(i).cuda(), torch.ones(len(u), dtype=torch.float64, device="cuda"), U, I)
    fit_phases(*args)
    gpu = fit_phases(*args)[3]
    res = dict(users=U, items=I, rows=len(u), gpu_fit_s=gpu["fit_s"])
    try:
        import sklearn  # noqa: F401
    except ImportError:
        res["reference"] = "not measured: sklearn is not installed"
        print("reference arm skipped: sklearn is not installed", file=sys.stderr)
        return res
    try:
        from oracle import ref_harness as rh
        rh.use_root(rh.INSTALLED_ROOT)
        if not rh.available():
            res["reference"] = "not measured: oracle/_ref absent"
            return res
        rh.import_reference()
        from daisy.model.PureSVDRecommender import PureSVD as RefPureSVD
        cfg = dict(gpu='0', logger=logging.getLogger('bench'), factors=FACTORS, topk=50, user_num=U, item_num=I,
                   optimizer='default', init_method='default', early_stop=False)
        m = RefPureSVD(cfg)
        df = pd.DataFrame({'user': u.astype(np.int64), 'item': i.astype(np.int64), 'rating': 1.0})
        t0 = time.perf_counter()
        m.fit(df)
        res["reference_fit_s"] = time.perf_counter() - t0
        res["host_cores"] = os.cpu_count()
    except Exception as e:  # noqa: BLE001
        res["reference"] = f"not measured: {e!r}"[:300]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="ml20m,netflix,transposed")
    ap.add_argument("--no-reference", action="store_true")
    a = ap.parse_args()
    ops.require_cuda()
    out = dict(bench="puresvd", factors=FACTORS, card=card())
    shapes = dict(ml20m=(138493, 26744, 20_000_263), netflix=(480189, 17770, 100_480_507),
                  transposed=(26744, 138493, 20_000_263))
    for w in a.workloads.split(","):
        out[w] = workload(*shapes[w])
        r = out[w]
        print(f"{w:>10}: fit {r['fit_s']:.3f} s | omega {r['omega_host_s']:.3f} csr {r['csr_s']:.3f} spmm {r['spmm_s']:.3f} "
              f"({r['spmm_calls']} x {r['spmm_ms_per_call']:.2f} ms, {r['spmm_tb_per_s']:.2f} TB/s algorithmic) orth "
              f"{r['orth_s']:.3f} small_svd {r['small_svd_s']:.3f} factors {r['factors_s']:.3f} | rank {r['rank_s'] * 1e3:.1f} ms "
              f"full_rank {r['full_rank_ms_per_user']:.3f} ms/user", file=sys.stderr)
    out["i8000"] = dict(status="not measured") if a.no_reference else reference_arm()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
