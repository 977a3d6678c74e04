"""Generates tests/golden/ease.npz from the reference's own EASE (daisy/model/EASERecommender.py), imported through
oracle/ref_harness.py.

Synthetic cases (B kept in full; the reference's rank on 30 candidates per user, full_rank and predict):
  c0  star values with duplicate (u, i) rows, a cold item, users without rows, reg 200
  c1  half-star values, reg 200                     (exact Gram, s = 1)
  c2  real-valued weights, reg 200                  (general fp64 Gram)
  c3  binary, I = 65 (no tile multiple), reg 3.5     (second reg value)
ml-100k on config 1's split (make_config("ease"): tsbr, reg 200, topk 50): digests of X and of the candidate sets, P's
diagonal (np.linalg.inv's own output, recorded during fit), rows 0, 1 and every 128th of B and B's column sums, rank on all
test users, full_rank of 4 users with train rows and 2 without, predict on 8 pairs, and the calc_ranking_results table.

    python oracle/gen_ease.py
"""
import hashlib
import os
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_harness as rh  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
B_STRIDE = 128                         # rows 0, 1 and every 128th row of the ml-100k B: the fixture stays under 300 KiB


def sha(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return np.frombuffer(h.digest(), np.uint8)


def _cases():
    rng = np.random.default_rng(21)
    out = []
    # c0: stars, 40 duplicated pairs with other values, item 44 cold, users 0 and 1 without rows
    u = rng.integers(2, 60, 700)
    i = rng.integers(0, 44, 700)
    k = rng.integers(0, 700, 40)
    u, i = np.concatenate([u, u[k]]), np.concatenate([i, i[k]])
    out.append(dict(U=60, I=45, reg=200.0, u=u, i=i, v=rng.integers(1, 6, len(u)).astype(np.float64)))
    u, i = rng.integers(0, 90, 1200), rng.integers(0, 60, 1200)
    out.append(dict(U=90, I=60, reg=200.0, u=u, i=i, v=rng.integers(1, 11, 1200) * 0.5))
    u, i = rng.integers(0, 150, 2000), rng.integers(0, 70, 2000)
    out.append(dict(U=150, I=70, reg=200.0, u=u, i=i, v=rng.random(2000) * 3.0 + 0.01))
    u, i = rng.integers(0, 80, 900), rng.integers(0, 65, 900)
    out.append(dict(U=80, I=65, reg=3.5, u=u, i=i, v=np.ones(900)))
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
    from daisy.model.EASERecommender import EASE
    rng = np.random.default_rng(5)
    cases = _cases()
    for k, c in enumerate(cases):
        df = pd.DataFrame({"user": c["u"].astype(np.int64), "item": c["i"].astype(np.int64), "rating": c["v"]})
        cfg = rh.make_config("ease", user_num=c["U"], item_num=c["I"], reg=c["reg"], topk=10, UID_NAME="user",
                             IID_NAME="item", INTER_NAME="rating")
        m = EASE(cfg)
        m.fit(df)
        users = np.arange(c["U"], dtype=np.int64)
        cands = np.stack([rng.choice(c["I"], 30, replace=False) for _ in users]).astype(np.int64)
        out[f"s{k}_u"], out[f"s{k}_i"], out[f"s{k}_v"] = c["u"].astype(np.int32), c["i"].astype(np.int32), c["v"]
        out[f"s{k}_meta"] = np.array([c["U"], c["I"], 10], np.int64)
        out[f"s{k}_reg"] = np.array(c["reg"], np.float64)
        out[f"s{k}_B"] = np.asarray(m.item_similarity, np.float64)
        out[f"s{k}_cands"] = cands.astype(np.int16)
        out[f"s{k}_rank"] = m.rank(_Loader(users, cands)).astype(np.int16)
        out[f"s{k}_full"] = np.concatenate([m.full_rank(int(u)) for u in users[:6]]).astype(np.int16)
        pi = cands[:, 0]
        out[f"s{k}_predict"] = np.array([m.predict(int(u), int(j)) for u, j in zip(users, pi)], np.float64)
    out["n_synthetic"] = np.array(len(cases))


def gen_ml100k(out):
    from daisy.model.EASERecommender import EASE
    from daisy.utils.dataset import CandidatesDataset, get_dataloader
    from daisy.utils.utils import build_candidates_set
    from daisy.utils.metrics import calc_ranking_results
    cfg = rh.make_config("ease")
    rh.seed_everything(cfg["seed"])
    art = rh.load_ml100k(cfg)
    train_set, test_ur, train_ur = art["train_set"], art["test_ur"], art["train_ur"]
    # config 1's split: the train rows of ml100k_sampler.npz, every value 1.0 (binary_inter)
    gs = np.load(os.path.join(GOLD, "ml100k_sampler.npz"))
    assert np.array_equal(train_set[cfg["UID_NAME"]].values, gs["coo_u"])
    assert np.array_equal(train_set[cfg["IID_NAME"]].values, gs["coo_i"])
    assert np.all(train_set[cfg["INTER_NAME"]].values == 1.0)
    model = EASE(cfg)                                              # test.py:8, 88
    inv, seen = np.linalg.inv, []

    def rec_inv(a):                                                # P as the reference's fit computes it
        p = inv(a)
        seen.append(np.asarray(p).copy())
        return p

    np.linalg.inv = rec_inv
    try:
        model.fit(train_set)                                       # test.py:95
    finally:
        np.linalg.inv = inv
    X, B = model.interaction_matrix, np.asarray(model.item_similarity)
    X.sort_indices()
    out["ml_meta"] = np.array([cfg["user_num"], cfg["item_num"], cfg["topk"], cfg["seed"], B_STRIDE], np.int64)
    out["ml_reg"] = np.array(cfg["reg"], np.float64)
    out["ml_X_sha"] = sha(X.indptr.astype(np.int64), X.indices.astype(np.int32), X.data.astype(np.float32))
    out["ml_P_diag"] = np.diag(seen[0]).copy()
    out["ml_B_rows"] = np.concatenate([B[:2], B[::B_STRIDE]])
    out["ml_B_colsum"] = B.sum(0)
    test_u, test_ucands = build_candidates_set(test_ur, train_ur, cfg)   # test.py:112
    cands = np.stack([c[1] for c in test_ucands]).astype(np.int64)
    out["ml_cands_sha"] = sha(cands)
    loader = get_dataloader(CandidatesDataset(test_ucands), batch_size=128, shuffle=False, num_workers=0)
    preds = model.rank(loader)                                     # test.py:120
    out["ml_test_u"] = np.array(test_u, np.int32)
    out["ml_rank"] = preds.astype(np.int16)
    warm = [u for u in test_u if X.indptr[u + 1] > X.indptr[u]][:4]
    cold = [u for u in test_u if X.indptr[u + 1] == X.indptr[u]][:2]
    out["ml_full_u"] = np.array(warm + cold, np.int32)
    out["ml_full"] = np.concatenate([model.full_rank(int(u)) for u in warm + cold]).astype(np.int16)
    pairs = np.array([[test_u[k], cands[k][-1 - k]] for k in range(8)], np.int64)
    out["ml_predict_pairs"] = pairs
    out["ml_predict"] = np.array([model.predict(int(u), int(i)) for u, i in pairs], np.float64)
    cfg["res_path"] = tempfile.mkdtemp() + "/"
    res = calc_ranking_results(test_ur, preds, test_u, cfg)        # test.py:131
    out["ml_kpi"] = res.values[:, 1:].astype(np.float64)
    out["ml_kpi_ks"] = np.array([int(c) for c in res.columns[1:]], np.int32)
    print(res)


def main():
    rh.import_reference()
    out = {}
    gen_synthetic(out)
    gen_ml100k(out)
    path = os.path.join(GOLD, "ease.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}  ({os.path.getsize(path) / 1024:.1f} KiB)")


if __name__ == "__main__":
    main()
