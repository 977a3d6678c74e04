"""EASE fit and scoring on one GPU; prints one JSON line.

Workloads (synthetic.make_interactions, seed 2022):
* ml20m_binary   the ML-20M shape (U = 138 493, I = 26 744, 20 M rows), binary values: the exact s8 Gram (s = 0);
* ml20m_half     the same rows with half-star values 0.5 .. 5: the exact Gram with s = 1;
* ml20m_real     the same rows with real-valued weights: the fp64 DMMA Gram;
* netflix_binary the Netflix shape (U = 480 189, I = 17 770, 100 M rows), binary.
The binary / real pair sits on both sides of the exact-path test, so both Gram kernels are measured.

Per workload: fit timed by phase (CSR, Gram, inverse, B) with device synchronisation around each phase; the Gram's rate in
TOPS over U * I * (I + 1) operations (a multiply and an add per lower-triangle product of the dense X^T X, the algorithmic
count, not the work done on the tiles), the inverse's in TFLOP/s over n^3 (the sweep operator's count on a symmetric matrix).
Then rank() for 4 096 users x 1 000 candidates and full_rank() per user (64 users in one call).
Reference arm: the reference's EASE.fit from oracle/_ref on the host cores at I = 8 000, beside the GPU at that shape.
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


def _sync_time(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in q.split(",")]
        return dict(name=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:  # noqa: BLE001
        return dict(name=torch.cuda.get_device_name(), power_limit=f"not read ({e!r})")


def fit_phases(d_u, d_i, d_v, U, I, reg=500.0):
    X, t_csr = _sync_time(lambda: ops.ease_csr(d_u, d_i, d_v, U, I))
    ws = ops.ease_workspace(X)
    G, t_gram = _sync_time(lambda: ops.ease_gram(X, reg, ws))
    _, t_inv = _sync_time(lambda: ops.ease_inverse(G, ws))
    _, t_b = _sync_time(lambda: ops.ease_weights(G, ws))
    return X, G, dict(scale=X.scale, csr_s=t_csr, gram_s=t_gram, inverse_s=t_inv, weights_s=t_b,
                      fit_s=t_csr + t_gram + t_inv + t_b,
                      gram_tops=U * I * (I + 1) / t_gram / 1e12, inverse_tflops=float(I) ** 3 / t_inv / 1e12)


def scoring(X, B, U, I, n_users=4096, n_cands=1000, n_full=64):
    g = torch.Generator(device="cuda")
    g.manual_seed(0)
    users = torch.randint(U, (n_users,), generator=g, device="cuda")
    cands = torch.randint(I, (n_users, n_cands), generator=g, device="cuda")
    ops.ease_rank(B, X, users, cands, 50)                     # warm-up
    _, t_rank = _sync_time(lambda: ops.ease_rank(B, X, users, cands, 50))
    fu = users[:n_full].contiguous()
    ops.ease_full_rank(B, X, fu, 50)
    _, t_full = _sync_time(lambda: ops.ease_full_rank(B, X, fu, 50))
    return dict(rank_s=t_rank, rank_users_per_s=n_users / t_rank, full_rank_ms_per_user=1e3 * t_full / n_full)


def workload(U, I, nnz, values):
    d = synthetic.make_interactions(U, I, nnz, device="cuda")
    d_u, d_i = d["coo_u"], d["coo_i"]
    n = d_u.numel()
    g = torch.Generator(device="cuda")
    g.manual_seed(1)
    if values == "binary":
        d_v = torch.ones(n, dtype=torch.float64, device="cuda")
    elif values == "half":
        d_v = torch.randint(1, 11, (n,), generator=g, device="cuda").to(torch.float64) * 0.5
    else:
        d_v = torch.rand(n, generator=g, device="cuda", dtype=torch.float64) * 4.0 + 0.5
    del d
    X, B, r = fit_phases(d_u, d_i, d_v, U, I)
    r.update(scoring(X, B, U, I))
    r.update(users=U, items=I, rows=n, values=values)
    del X, B
    torch.cuda.empty_cache()
    return r


def reference_arm(U=40000, I=8000, nnz=2_000_000):
    """The reference's EASE.fit (numpy / scipy on the host) and the GPU fit on the same rows."""
    import pandas as pd
    d = synthetic.make_interactions(U, I, nnz, device="cpu")
    u, i = d["coo_u"].numpy(), d["coo_i"].numpy()
    gpu = fit_phases(torch.from_numpy(u).cuda(), torch.from_numpy(i).cuda(), torch.ones(len(u), dtype=torch.float64,
                                                                                           device="cuda"), U, I)[2]
    res = dict(users=U, items=I, rows=len(u), gpu_fit_s=gpu["fit_s"])
    try:
        from oracle import ref_harness as rh
        rh.use_root(rh.INSTALLED_ROOT)
        if not rh.available():
            res["reference"] = "not measured: oracle/_ref absent"
            return res
        rh.import_reference()
        from daisy.model.EASERecommender import EASE as RefEASE
        cfg = dict(gpu='0', logger=logging.getLogger('bench'), reg=500.0, topk=50, user_num=U, item_num=I, UID_NAME='user',
                   IID_NAME='item', INTER_NAME='rating', optimizer='default', init_method='default', early_stop=False)
        m = RefEASE(cfg)
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
    ap.add_argument("--workloads", default="ml20m_binary,ml20m_half,ml20m_real,netflix_binary")
    ap.add_argument("--no-reference", action="store_true")
    a = ap.parse_args()
    ops.require_cuda()
    out = dict(bench="ease", card=card())
    d = synthetic.make_interactions(2000, 700, 40000, device="cuda")          # loads every kernel before the timed runs
    X, B, _ = fit_phases(d["coo_u"], d["coo_i"], torch.ones(d["coo_u"].numel(), dtype=torch.float64, device="cuda"), 2000, 700)
    scoring(X, B, 2000, 700)
    fit_phases(d["coo_u"], d["coo_i"], torch.rand(d["coo_u"].numel(), dtype=torch.float64, device="cuda"), 2000, 700)
    shapes = dict(ml20m_binary=(138493, 26744, 20_000_263, "binary"), ml20m_half=(138493, 26744, 20_000_263, "half"),
                  ml20m_real=(138493, 26744, 20_000_263, "real"), netflix_binary=(480189, 17770, 100_480_507, "binary"))
    for w in a.workloads.split(","):
        out[w] = workload(*shapes[w])
    out["reference_arm"] = dict(status="not measured") if a.no_reference else reference_arm()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
