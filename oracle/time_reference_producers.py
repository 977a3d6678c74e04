"""Time the REFERENCE's own host-side producers / consumers of the hot path on this machine's CPU (build container only:
imports /root/reference through oracle/ref_harness.py).  TEST INFRASTRUCTURE -- gives the CPU side of the section-8(f)
rows whose GPU side is bench.py's configs.inference / sampling / shuffle lines.  Shapes are cut down where the reference is O(U * I) in Python and
the full-size time is extrapolated linearly in the number of users (stated in the output).

    python -m oracle.time_reference_producers
"""
import json
import logging
import os
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_harness as rh  # noqa: E402


def main():
    rh.import_reference()
    import pandas as pd
    from daisy.utils.metrics import calc_ranking_results
    from daisy.utils.sampler import BasicNegtiveSampler
    from daisy.utils.utils import get_ur, get_inter_matrix
    rng = np.random.default_rng(0)
    out = {"machine": {"cpus": os.cpu_count()}}

    # ---- KPIs: calc_ranking_results on n users x top-50 (ML-20M item count), 5 default metrics x 6 cut-offs
    I, K = 26744, 50
    for n in (5000, 20000):
        test_u = list(range(n))
        test_ur = {u: set(rng.integers(0, I, size=int(rng.integers(1, 21))).tolist()) for u in test_u}
        preds = rng.integers(0, I, size=(n, K)).astype(np.float32)
        cfg = {"logger": logging.getLogger("t"), "res_path": tempfile.mkdtemp() + "/", "metrics": ["recall", "mrr", "ndcg", "hit", "precision"],
               "item_num": I, "topk": K}
        t0 = time.perf_counter()
        calc_ranking_results(test_ur, preds, test_u, cfg)
        dt = time.perf_counter() - t0
        out[f"kpis_{n}_users_s"] = dt
    out["kpis_138493_users_extrapolated_s"] = out["kpis_20000_users_s"] * 138493 / 20000

    # ---- sampler: per-user setdiff1d over the item range (ML-20M item count), 2 000 users, 145 interactions each
    U, G = 2000, 4
    cu = np.repeat(np.arange(U), 145)
    ci = rng.integers(0, I, size=len(cu))
    df = pd.DataFrame({"user": cu, "item": ci, "rating": 1.0, "timestamp": np.arange(len(cu))})
    t0 = time.perf_counter()
    ur = get_ur(df)
    out["get_ur_290k_rows_s"] = time.perf_counter() - t0
    cfg = rh.make_config("mf", user_num=U, item_num=I, num_ng=G, train_ur=ur)
    np.random.seed(1)
    t0 = time.perf_counter()
    BasicNegtiveSampler(df, cfg).sampling()
    dt = time.perf_counter() - t0
    out["sampling_2000_users_s"] = dt
    out["sampling_138493_users_extrapolated_s"] = dt * 138493 / U
    out["get_ur_20M_rows_extrapolated_s"] = out["get_ur_290k_rows_s"] * 20_000_000 / len(cu)

    # ---- LightGCN adjacency: dok_matrix update + D A D on 300 k interactions (Amazon-Book node counts)
    import torch
    from daisy.model.LightGCNRecommender import LightGCN
    U4, I4, nnz = 52643, 91599, 300_000
    cu = rng.integers(0, U4, size=nnz)
    ci = rng.integers(0, I4, size=nnz)
    df = pd.DataFrame({"user": cu, "item": ci, "rating": 1.0, "timestamp": np.arange(nnz)})
    cfg = rh.make_config("lightgcn", user_num=U4, item_num=I4, factors=8, num_layers=1)
    t0 = time.perf_counter()
    cfg["inter_matrix"] = get_inter_matrix(df, cfg)
    torch.manual_seed(0)
    LightGCN(cfg)                                          # get_norm_adj_mat runs in the constructor (:70)
    dt = time.perf_counter() - t0
    out["lightgcn_adjacency_300k_edges_s"] = dt
    out["lightgcn_adjacency_3M_edges_extrapolated_s"] = dt * 10
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
