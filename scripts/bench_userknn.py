"""UserKNNCF and MostPop on the GPU path at the ML-20M shape (138 493 users, 26 744 items, 20 000 263 rows, item ids
Zipf-distributed): UserKNN fit split into its phases (CSR, transform, image, Gram, selection, reverse lists), binary and
half-star values, with tensor TOPS over 2 U^2 I for the Gram; rank of 4 096 users x 1 000 candidates and full_rank per user;
MostPop fit and rank at the same shape.  Prints one JSON line with the card's name and power limit read in the same run.

    python scripts/bench_userknn.py [--maxk 100]
"""
import argparse
import json
import logging
import os
import subprocess
import sys
import time

import numpy as np
import pandas as pd
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from daisyrec_b200 import ops  # noqa: E402
from daisyrec_b200.model import MostPop, UserKNNCF  # noqa: E402

U, I, NNZ = 138493, 26744, 20_000_263


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                            text=True, timeout=20).stdout.strip()
    except Exception:                                  # noqa: BLE001
        pl = "not measured"
    return name, pl


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, time.perf_counter() - t


def fit_phases(u, i, v, maxk):
    d = lambda a, t: torch.from_numpy(np.ascontiguousarray(a, t)).cuda()
    d_u, d_i, d_v = d(u, np.int32), d(i, np.int32), d(v, np.float64)
    out = {}
    X, out['csr_s'] = timed(lambda: ops.ease_csr(d_u, d_i, d_v, U, I))
    (Xt, ss), out['transform_s'] = timed(lambda: ops.userknn_transform(X, d_u, d_i, 'cosine'))
    img, out['image_s'] = timed(lambda: ops.gram_image(Xt))
    free = torch.cuda.mem_get_info()[0]
    panel = ops.userknn_panel_rows(U, free - 24 * U * maxk - (1 << 30))
    n = Xt.item_num
    idx = torch.empty((n, maxk), dtype=torch.int32, device='cuda')
    val = torch.empty((n, maxk), dtype=torch.float32, device='cuda')
    cnt = torch.empty(n, dtype=torch.int32, device='cuda')
    buf = torch.empty(min(panel, n) * n, dtype=torch.float64, device='cuda')
    gram = sel = 0.0
    for p0 in range(0, n, panel):
        r = min(panel, n - p0)
        G, t = timed(lambda: ops.gram_panel(img, Xt, p0, r, buf))
        gram += t
        _, t = timed(lambda: ops.L.check(ops.L.lib().drb_knn_neighbours_panel(
            ops._ptr(G), n, p0, r, ops._ptr(ss), 0, 1, 100.0, maxk, ops._ptr(idx), ops._ptr(val), ops._ptr(cnt), ops._stream())))
        sel += t
    out.update(gram_s=gram, select_s=sel, panel_rows=panel, exact=Xt.scale >= 0, gram_tops=2.0 * U * U * I / gram / 1e12)
    del img, buf
    _, out['reverse_s'] = timed(lambda: ops.userknn_reverse(ops.KnnNeighbours(idx, val, cnt)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--maxk', type=int, default=100)
    a = ap.parse_args()
    rng = np.random.default_rng(0)
    u = rng.integers(0, U, NNZ)
    i = np.minimum(rng.zipf(1.3, NNZ) - 1, I - 1)
    res = {'shape': [U, I, NNZ], 'maxk': a.maxk}
    name, pl = card()
    res['card'], res['power_limit'] = name, pl
    res['binary'] = fit_phases(u, i, np.ones(NNZ), a.maxk)
    torch.cuda.empty_cache()
    res['half_star'] = fit_phases(u, i, rng.integers(1, 11, NNZ) * 0.5, a.maxk)
    torch.cuda.empty_cache()
    m = UserKNNCF(dict(user_num=U, item_num=I, maxk=a.maxk, shrink=100, normalize=True, similarity='cosine', topk=50,
                       logger=logging.getLogger('b')))
    df = pd.DataFrame({'user': u, 'item': i, 'rating': np.ones(NNZ)})
    _, res['fit_binary_s'] = timed(lambda: m.fit(df))
    users = torch.from_numpy(rng.choice(U, 4096, replace=False)).cuda()
    cands = torch.from_numpy(rng.integers(0, I, (4096, 1000))).cuda()
    ops.userknn_rank(m._X, m._R, users, cands, 50)
    _, res['rank_4096x1000_s'] = timed(lambda: ops.userknn_rank(m._X, m._R, users, cands, 50))
    m.full_rank(1)
    _, t = timed(lambda: [m.full_rank(int(x)) for x in range(64)])
    res['full_rank_per_user_s'] = t / 64
    del m
    torch.cuda.empty_cache()
    p = MostPop(dict(item_num=I, topk=50, IID_NAME='item', logger=logging.getLogger('b')))
    p.fit(df)
    _, res['mostpop_fit_s'] = timed(lambda: p.fit(df))
    d_cands = cands
    ops.mostpop_rank(p._score, d_cands, 50)
    _, res['mostpop_rank_4096x1000_s'] = timed(lambda: ops.mostpop_rank(p._score, d_cands, 50))
    print(json.dumps(res))


if __name__ == '__main__':
    main()
