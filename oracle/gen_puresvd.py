"""Generates tests/golden/puresvd.npz from the reference's own PureSVD (daisy/model/PureSVDRecommender.py), imported through
oracle/ref_harness.py.

Synthetic cases (user_vec, item_vec and sigma in full; the reference's rank on 30 candidates per user, full_rank of 6 users and
predict on one pair per user):
  s0  U >= I, factors < 0.1 min(U, I): the non-transposed branch, n_iter 7
  s1  U < I, factors >= 0.1 min(U, I): the transposed branch, n_iter 4
  s2  star values with duplicate (u, i) rows, cold users and a cold item
  s3  real-valued weights, each an fp32 number (transposed, n_iter 7)
  s4  factors + 10 == min(U, I), every user and item with rows
  s5  rank(X) < factors + 10 (15 distinct user rows): only the data, for the device's refusal
ml-100k on config 1's split with puresvd.yaml (factors 150): X's digest, sigma, rows 0, 1 and every 8th of user_vec and
item_vec and their column sums, the candidate digest, rank on all test users with their warm / cold mask, full_rank of 4 warm
users, predict on 8 pairs, the calc_ranking_results table, and the same table after the cold users' rows are replaced by the
first topk candidates (what exact zero factor rows give).

    python oracle/gen_puresvd.py
"""
import hashlib
import os
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_harness as rh  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
ROW_STRIDE = 8


def sha(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return np.frombuffer(h.digest(), np.uint8)


def _cases():
    rng = np.random.default_rng(2019)
    out = []
    u, i = rng.integers(0, 150, 1800), rng.integers(0, 100, 1800)
    out.append(dict(U=150, I=100, factors=8, u=u, i=i, v=np.ones(len(u))))
    u, i = rng.integers(0, 40, 1600), rng.integers(0, 100, 1600)
    out.append(dict(U=40, I=100, factors=12, u=u, i=i, v=rng.integers(1, 6, len(u)).astype(np.float64)))
    # users 0..3 and item 79 cold, 150 duplicated pairs with their own values
    u, i = rng.integers(4, 100, 1500), rng.integers(0, 79, 1500)
    k = rng.integers(0, 1500, 150)
    u, i = np.concatenate([u, u[k]]), np.concatenate([i, i[k]])
    out.append(dict(U=100, I=80, factors=5, u=u, i=i, v=rng.integers(1, 6, len(u)).astype(np.float64)))
    u, i = rng.integers(0, 80, 2000), rng.integers(0, 140, 2000)
    out.append(dict(U=80, I=140, factors=5, u=u, i=i, v=(rng.random(len(u)) * 3.0 + 0.01).astype(np.float32).astype(np.float64)))
    # dense enough for full column rank; every user and item has rows
    mask = rng.random((50, 30)) < 0.5
    mask[np.arange(50), np.arange(50) % 30] = True
    u, i = np.nonzero(mask)
    out.append(dict(U=50, I=30, factors=20, u=u, i=i, v=rng.integers(1, 6, len(u)).astype(np.float64)))
    # 15 distinct user rows: rank(X) <= 15 < l = 20
    base = rng.random((15, 70)) < 0.3
    rows = base[rng.integers(0, 15, 80)]
    rows[:15] = base
    u, i = np.nonzero(rows)
    out.append(dict(U=80, I=70, factors=10, u=u, i=i, v=np.ones(len(u)), deficient=True))
    return out


class _Loader:
    """(us, cands_ids) batches, as the reference's rank iterates its test loader."""

    def __init__(self, users, cands, bs=16):
        self.users, self.cands, self.bs = users, cands, bs

    def __iter__(self):
        import torch
        for s in range(0, len(self.users), self.bs):
            yield torch.from_numpy(self.users[s:s + self.bs]), torch.from_numpy(self.cands[s:s + self.bs])


def gen_synthetic(out):
    import pandas as pd
    import sklearn.utils.extmath as ext
    from daisy.model.PureSVDRecommender import PureSVD
    from oracle import puresvd_oracle as po
    rng = np.random.default_rng(5)
    cases = _cases()
    for k, c in enumerate(cases):
        U, I, f = c["U"], c["I"], c["factors"]
        X = po.interaction_matrix(c["u"], c["i"], c["v"], U, I)
        l = f + 10
        assert (np.linalg.matrix_rank(X.toarray()) < l) == bool(c.get("deficient")), k
        out[f"s{k}_u"], out[f"s{k}_i"] = c["u"].astype(np.int16), c["i"].astype(np.int16)
        out[f"s{k}_v"] = c["v"].astype(np.float32)          # every value is an fp32 number: stored without loss
        out[f"s{k}_meta"] = np.array([U, I, f, 10, int(bool(c.get("deficient")))], np.int64)
        if c.get("deficient"):
            continue
        df = pd.DataFrame({"user": c["u"].astype(np.int64), "item": c["i"].astype(np.int64), "rating": c["v"]})
        cfg = rh.make_config("puresvd", user_num=U, item_num=I, factors=f, topk=10)
        m = PureSVD(cfg)
        seen = []
        rs = ext.randomized_svd

        def rec(*a, **kw):                                         # sigma as the reference's fit computes it
            r = rs(*a, **kw)
            seen.append(r[1].copy())
            return r

        import daisy.model.PureSVDRecommender as mod
        mod.randomized_svd = rec
        try:
            m.fit(df)
        finally:
            mod.randomized_svd = rs
        users = np.arange(U, dtype=np.int64)
        cands = np.stack([rng.choice(I, 30, replace=False) for _ in users]).astype(np.int64)
        out[f"s{k}_user_vec"] = np.asarray(m.user_vec, np.float64)
        out[f"s{k}_item_vec"] = np.asarray(m.item_vec, np.float64)
        out[f"s{k}_sigma"] = seen[0]
        out[f"s{k}_cands"] = cands.astype(np.int16)
        out[f"s{k}_rank"] = m.rank(_Loader(users, cands)).astype(np.int16)
        warm = [a for a in users if X.indptr[a + 1] > X.indptr[a]][:6]
        out[f"s{k}_full_u"] = np.array(warm, np.int32)
        out[f"s{k}_full"] = np.stack([m.full_rank(int(a)) for a in warm]).astype(np.int16)
        out[f"s{k}_predict"] = np.array([m.predict(int(a), int(j)) for a, j in zip(users, cands[:, 0])], np.float64)
    out["n_synthetic"] = np.array(len(cases))


def gen_ml100k(out):
    import sklearn.utils.extmath as ext
    import daisy.model.PureSVDRecommender as mod
    from daisy.model.PureSVDRecommender import PureSVD
    from daisy.utils.dataset import CandidatesDataset, get_dataloader
    from daisy.utils.utils import build_candidates_set
    from daisy.utils.metrics import calc_ranking_results
    cfg = rh.make_config("puresvd")
    rh.seed_everything(cfg["seed"])
    art = rh.load_ml100k(cfg)
    train_set, test_ur, train_ur = art["train_set"], art["test_ur"], art["train_ur"]
    gs = np.load(os.path.join(GOLD, "ml100k_sampler.npz"))
    assert np.array_equal(train_set["user"].values, gs["coo_u"])
    assert np.array_equal(train_set["item"].values, gs["coo_i"])
    assert np.all(train_set["rating"].values == 1.0)
    model = PureSVD(cfg)                                           # test.py:75-76
    seen, rs = [], ext.randomized_svd

    def rec(*a, **kw):
        r = rs(*a, **kw)
        seen.append(r[1].copy())
        return r

    mod.randomized_svd = rec
    try:
        model.fit(train_set)
    finally:
        mod.randomized_svd = rs
    U, I = cfg["user_num"], cfg["item_num"]
    X = model._convert_df(U, I, train_set)
    X.sum_duplicates()
    X.sort_indices()
    P, Qv = np.asarray(model.user_vec), np.asarray(model.item_vec)
    out["ml_meta"] = np.array([U, I, cfg["topk"], cfg["seed"], ROW_STRIDE, cfg["factors"]], np.int64)
    out["ml_X_sha"] = sha(X.indptr.astype(np.int64), X.indices.astype(np.int32), X.data.astype(np.float64))
    out["ml_sigma"] = seen[0]
    out["ml_user_rows"] = np.concatenate([P[:2], P[::ROW_STRIDE]])
    out["ml_item_rows"] = np.concatenate([Qv[:2], Qv[::ROW_STRIDE]])
    out["ml_user_colsum"] = P.sum(0)
    out["ml_item_colsum"] = Qv.sum(0)
    test_u, test_ucands = build_candidates_set(test_ur, train_ur, cfg)   # test.py:112
    cands = np.stack([c[1] for c in test_ucands]).astype(np.int64)
    out["ml_cands_sha"] = sha(cands)
    loader = get_dataloader(CandidatesDataset(test_ucands), batch_size=128, shuffle=False, num_workers=0)
    preds = model.rank(loader)                                     # test.py:120
    warm = np.diff(X.indptr)[np.asarray(test_u)] > 0
    out["ml_test_u"] = np.array(test_u, np.int32)
    out["ml_rank"] = preds.astype(np.int16)
    out["ml_warm"] = warm
    wu = [u for u, w in zip(test_u, warm) if w][:4]
    out["ml_full_u"] = np.array(wu, np.int32)
    out["ml_full"] = np.stack([model.full_rank(int(u)) for u in wu]).astype(np.int16)
    pairs = np.array([[test_u[k], cands[k][-1 - k]] for k in range(8)], np.int64)
    out["ml_predict_pairs"] = pairs
    out["ml_predict"] = np.array([model.predict(int(u), int(i)) for u, i in pairs], np.float64)
    cfg["res_path"] = tempfile.mkdtemp() + "/"
    res = calc_ranking_results(test_ur, preds, test_u, cfg)        # test.py:131
    out["ml_kpi"] = res.values[:, 1:].astype(np.float64)
    out["ml_kpi_ks"] = np.array([int(c) for c in res.columns[1:]], np.int32)
    sub = preds.copy()
    sub[~warm] = cands[~warm, :cfg["topk"]]
    res_sub = calc_ranking_results(test_ur, sub, test_u, cfg)
    out["ml_kpi_sub"] = res_sub.values[:, 1:].astype(np.float64)
    print(res)
    print(res_sub)


def main():
    rh.import_reference()
    out = {}
    gen_synthetic(out)
    gen_ml100k(out)
    path = os.path.join(GOLD, "puresvd.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}  ({os.path.getsize(path) / 1024:.1f} KiB)")


if __name__ == "__main__":
    main()
