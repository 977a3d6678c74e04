"""SLiM fit on one GPU; prints one JSON line.

Workloads, binary values:
* ml100k          config 1's ml-100k split (tests/golden/ml100k_sampler.npz) at assets/slim.yaml, alpha 1.0, elastic 0.1;
* ml20m_binary    the ML-20M shape (U = 138 493, I = 26 744, 20 M rows; synthetic.make_interactions, seed 2022);
* netflix_binary  the Netflix shape (U = 480 189, I = 17 770, 100 M rows);
the synthetic shapes at (alpha, elastic) = (1.0, 0.1) and (0.1, 0.1), topk 50, sklearn's tol 1e-4 and max_iter 100.

Per workload and configuration, after a warm-up fit at the same shape: the fit timed by phase with device events (CSR, Gram,
live lists, solve, selection), the sweeps (mean and max over items), the live fraction (live coordinates over I (I - 1)), the
largest live list, and how many items stopped at max_iter.
Reference arm (only when the installed reference copy in oracle/_ref and sklearn import): the reference's per-item loop body
(SLiMRecommender.py:74-109, its own ElasticNet instance) timed on 24 sampled items at I = 8 000 (40 000 users, 2 M rows), and
the full fit extrapolated from it, beside the GPU fit at that shape.
"""
import argparse
import json
import logging
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from daisyrec_b200 import ops  # noqa: E402
from daisyrec_b200.utils import synthetic  # noqa: E402
from scripts.bench_ease import card  # noqa: E402
from scripts.bench_itemknn import _event_time  # noqa: E402

CONFIGS = ((1.0, 0.1), (0.1, 0.1))


def fit_phases(d_u, d_i, d_v, U, I, alpha, elastic, topk=50, tol=1e-4, max_iter=100):
    X, t_csr = _event_time(lambda: ops.ease_csr(d_u, d_i, d_v, U, I))
    ws = ops.ease_workspace(X)
    G, t_gram = _event_time(lambda: ops.ease_gram(X, 0.0, ws))
    del ws
    l1, l2 = alpha * elastic * U, alpha * (1.0 - elastic) * U
    P, t_live = _event_time(lambda: ops.slim_live(G, l1))
    P, t_solve = _event_time(lambda: ops.slim_solve(G, l1, l2, tol, max_iter, panel=P))
    W, t_sel = _event_time(lambda: ops.slim_select(P, topk))
    nl = P.nl.double()
    sweeps = P.sweeps.double()
    r = dict(alpha=alpha, elastic=elastic, csr_s=t_csr, gram_s=t_gram, live_s=t_live, solve_s=t_solve, select_s=t_sel,
             fit_s=t_csr + t_gram + t_live + t_solve + t_sel, sweeps_mean=float(sweeps.mean()), sweeps_max=int(sweeps.max()),
             live_fraction=float(nl.sum()) / (I * max(I - 1, 1)), live_max=int(nl.max()),
             stopped_at_max_iter=int((P.conv == 0).sum()), neighbours=int(W.cnt.sum()))
    del P, G
    return X, W, r


def workload(d_u, d_i, U, I, configs):
    d_u, d_i = d_u.to(torch.int32).contiguous(), d_i.to(torch.int32).contiguous()
    d_v = torch.ones(d_u.numel(), dtype=torch.float64, device="cuda")
    out = dict(users=U, items=I, rows=d_u.numel())
    for alpha, elastic in configs:
        fit_phases(d_u, d_i, d_v, U, I, alpha, elastic)                       # warm-up fit
        torch.cuda.empty_cache()
        _, _, r = fit_phases(d_u, d_i, d_v, U, I, alpha, elastic)
        torch.cuda.empty_cache()
        out[f"a{alpha}_e{elastic}"] = r
    return out


def reference_arm(U=40000, I=8000, nnz=2_000_000, n_cols=24, alpha=1.0, elastic=0.1):
    d = synthetic.make_interactions(U, I, nnz, device="cpu")
    u, i = d["coo_u"].numpy(), d["coo_i"].numpy()
    res = workload(torch.from_numpy(u).cuda(), torch.from_numpy(i).cuda(), U, I, ((alpha, elastic),))
    try:
        import pandas as pd
        import sklearn  # noqa: F401
        from oracle import ref_harness as rh
        rh.use_root(rh.INSTALLED_ROOT)
        if not rh.available():
            res["reference"] = "not measured: oracle/_ref absent"
            return res
        rh.import_reference()
        from daisy.model.SLiMRecommender import SLiM as RefSLiM
        cfg = dict(gpu='', logger=logging.getLogger('bench'), alpha=alpha, elastic=elastic, topk=50, user_num=U, item_num=I,
                   optimizer='default', init_method='default', early_stop=False)
        m = RefSLiM(cfg)
        train = m._convert_df(U, I, pd.DataFrame({'user': u.astype(np.int64), 'item': i.astype(np.int64), 'rating': 1.0}))
        cols = np.random.default_rng(0).choice(I, n_cols, replace=False)
        t0 = time.perf_counter()
        for j in cols:                                  # SLiMRecommender.py:74-109 for item j
            y = train[:, j].toarray()
            s, e = train.indptr[j], train.indptr[j + 1]
            backup = train.data[s:e].copy()
            train.data[s:e] = 0.0
            m.md.fit(train, y)
            _ = m.md.sparse_coef_
            train.data[s:e] = backup
        per = (time.perf_counter() - t0) / n_cols
        res["reference_s_per_item"] = per
        res["reference_fit_s_extrapolated"] = per * I
        res["reference_items_sampled"] = n_cols
        res["host_cores"] = os.cpu_count()
    except Exception as e:  # noqa: BLE001
        res["reference"] = f"not measured: {e!r}"[:300]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="ml100k,ml20m_binary,netflix_binary")
    ap.add_argument("--no-reference", action="store_true")
    a = ap.parse_args()
    ops.require_cuda()
    out = dict(bench="slim", card=card())
    shapes = dict(ml20m_binary=(138493, 26744, 20_000_263), netflix_binary=(480189, 17770, 100_480_507))
    for w in a.workloads.split(","):
        if w == "ml100k":
            gs = np.load(os.path.join(ROOT, "tests", "golden", "ml100k_sampler.npz"))
            cu, ci = gs["coo_u"].astype(np.int64), gs["coo_i"].astype(np.int64)
            U, I = int(cu.max()) + 1, int(ci.max()) + 1
            out[w] = workload(torch.from_numpy(cu).cuda(), torch.from_numpy(ci).cuda(), U, I, ((1.0, 0.1),))
        else:
            d = synthetic.make_interactions(*shapes[w], device="cuda")
            out[w] = workload(d["coo_u"], d["coo_i"], shapes[w][0], shapes[w][1], CONFIGS)
            del d
        torch.cuda.empty_cache()
    out["reference_arm"] = dict(status="not measured") if a.no_reference else reference_arm()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
