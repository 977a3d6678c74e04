"""ItemKNNCF fit and scoring on one GPU; prints one JSON line.

Workloads (synthetic.make_interactions, seed 2022), cosine with shrink 100 and maxk 40 (assets/itemknn.yaml):
* ml20m_binary    the ML-20M shape (U = 138 493, I = 26 744, 20 M rows), binary values: the exact s8 Gram;
* netflix_binary  the Netflix shape (U = 480 189, I = 17 770, 100 M rows), binary.

Per workload, after a warm-up fit at the same shape: fit timed by phase (CSR, value transform + scale decision, Gram, neighbour
selection) with device events; the selection kernel's read rate, 8 I^2 bytes of G over its time, beside the 3.35 TB/s of the
H100 SXM data sheet (the kernel re-reads each row of G four times, from L2 when it stays there, so this is a rate over the
bytes the algorithm needs, not a share of peak).  Then rank() for 4 096 users x 1 000 candidates and full_rank() per user (64
users in one call).
Reference arm: the reference's ItemKNNCF.fit from oracle/_ref on the host cores at I = 8 000, beside the GPU at that shape.
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

HBM_BYTES_PER_S = 3.35e12


def _event_time(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    b.synchronize()
    return out, a.elapsed_time(b) / 1e3


def fit_phases(d_u, d_i, d_v, U, I, similarity="cosine", normalize=True, shrink=100, maxk=40):
    X, t_csr = _event_time(lambda: ops.ease_csr(d_u, d_i, d_v, U, I))
    (Xt, ss, _), t_tr = _event_time(lambda: ops.itemknn_transform(X, similarity))
    ws = ops.ease_workspace(Xt)
    G, t_gram = _event_time(lambda: ops.ease_gram(Xt, 0.0, ws))
    W, t_sel = _event_time(lambda: ops.itemknn_neighbours(G, ss, similarity, normalize, shrink, maxk))
    return X, W, dict(scale=Xt.scale, csr_s=t_csr, transform_s=t_tr, gram_s=t_gram, select_s=t_sel,
                      fit_s=t_csr + t_tr + t_gram + t_sel, select_gram_bytes_per_s=8.0 * I * I / t_sel,
                      select_rate_over_hbm_datasheet=8.0 * I * I / t_sel / HBM_BYTES_PER_S)


def scoring(X, W, U, I, n_users=4096, n_cands=1000, n_full=64):
    g = torch.Generator(device="cuda")
    g.manual_seed(0)
    users = torch.randint(U, (n_users,), generator=g, device="cuda")
    cands = torch.randint(I, (n_users, n_cands), generator=g, device="cuda")
    ops.itemknn_rank(X, W, users, cands, 50)                     # warm-up
    _, t_rank = _event_time(lambda: ops.itemknn_rank(X, W, users, cands, 50))
    fu = users[:n_full].contiguous()
    ops.itemknn_full_rank(X, W, fu, 50)
    _, t_full = _event_time(lambda: ops.itemknn_full_rank(X, W, fu, 50))
    return dict(rank_s=t_rank, rank_users_per_s=n_users / t_rank, full_rank_ms_per_user=1e3 * t_full / n_full)


def workload(U, I, nnz):
    d = synthetic.make_interactions(U, I, nnz, device="cuda")
    d_u, d_i = d["coo_u"], d["coo_i"]
    d_v = torch.ones(d_u.numel(), dtype=torch.float64, device="cuda")
    del d
    fit_phases(d_u, d_i, d_v, U, I)                              # warm-up fit
    torch.cuda.empty_cache()
    X, W, r = fit_phases(d_u, d_i, d_v, U, I)
    r.update(scoring(X, W, U, I))
    r.update(users=U, items=I, rows=d_u.numel(), neighbours=int(W.cnt.sum()))
    del X, W
    torch.cuda.empty_cache()
    return r


def reference_arm(U=40000, I=8000, nnz=2_000_000):
    """The reference's ItemKNNCF.fit (numpy / scipy on the host) and the GPU fit on the same rows."""
    import pandas as pd
    d = synthetic.make_interactions(U, I, nnz, device="cpu")
    u, i = d["coo_u"].numpy(), d["coo_i"].numpy()
    args = (torch.from_numpy(u).cuda(), torch.from_numpy(i).cuda(), torch.ones(len(u), dtype=torch.float64, device="cuda"), U, I)
    fit_phases(*args)
    res = dict(users=U, items=I, rows=len(u), gpu_fit_s=fit_phases(*args)[2]["fit_s"])
    try:
        from oracle import ref_harness as rh
        rh.use_root(rh.INSTALLED_ROOT)
        if not rh.available():
            res["reference"] = "not measured: oracle/_ref absent"
            return res
        rh.import_reference()
        from daisy.model.KNNCFRecommender import ItemKNNCF as RefItemKNN
        cfg = dict(gpu='0', logger=logging.getLogger('bench'), maxk=40, shrink=100, normalize=True, similarity='cosine', topk=50,
                   user_num=U, item_num=I, optimizer='default', init_method='default', early_stop=False)
        m = RefItemKNN(cfg)
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
    ap.add_argument("--workloads", default="ml20m_binary,netflix_binary")
    ap.add_argument("--no-reference", action="store_true")
    a = ap.parse_args()
    ops.require_cuda()
    out = dict(bench="itemknn", card=card())
    shapes = dict(ml20m_binary=(138493, 26744, 20_000_263), netflix_binary=(480189, 17770, 100_480_507))
    for w in a.workloads.split(","):
        out[w] = workload(*shapes[w])
    out["reference_arm"] = dict(status="not measured") if a.no_reference else reference_arm()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
