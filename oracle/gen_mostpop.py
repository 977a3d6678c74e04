"""Generates tests/golden/mostpop.npz from the reference's own MostPop (daisy/model/PopRecommender.py), imported through
oracle/ref_harness.py with gen_itemknn.py's shims.

A synthetic set (duplicate rows, items without rows, many equal counts) and ml-100k on config 1's split with
assets/mostpop.yaml: item_cnt_ref and item_score in full, rank on all test users (the reference's float32 ids), full_rank,
predict and the KPI table.  The reference orders equal scores with unstable sorts, so the ids inside a tie group are only
what it happened to return.

    python oracle/gen_mostpop.py
"""
import os
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_harness as rh  # noqa: E402
from oracle.gen_itemknn import GOLD, _Loader, _shims  # noqa: E402


def gen_synthetic(out):
    import pandas as pd
    from daisy.model.PopRecommender import MostPop
    rng = np.random.default_rng(8)
    U, I = 50, 40
    i = rng.integers(0, 30, 400)
    u = rng.integers(0, U, 400)
    df = pd.DataFrame({"user": u, "item": i, "rating": np.ones(400)})
    cfg = rh.make_config("mostpop", user_num=U, item_num=I, topk=10)
    m = MostPop(cfg)
    m.fit(df)
    users = np.arange(U, dtype=np.int64)
    cands = np.stack([rng.choice(I, 25, replace=False) for _ in users]).astype(np.int64)
    out["s_u"], out["s_i"], out["s_meta"], out["s_cands"] = u.astype(np.int16), i.astype(np.int16), np.array([U, I, 10]), cands
    out["s_cnt"], out["s_score"] = m.item_cnt_ref, m.item_score
    out["s_rank"] = m.rank(_Loader(users, cands))
    out["s_full"] = m.full_rank(0)


def gen_ml100k(out):
    from daisy.model.PopRecommender import MostPop
    from daisy.utils.dataset import CandidatesDataset, get_dataloader
    from daisy.utils.utils import build_candidates_set
    from daisy.utils.metrics import calc_ranking_results
    cfg = rh.make_config("mostpop")
    rh.seed_everything(cfg["seed"])
    art = rh.load_ml100k(cfg)
    train_set, test_ur, train_ur = art["train_set"], art["test_ur"], art["train_ur"]
    gs = np.load(os.path.join(GOLD, "ml100k_sampler.npz"))
    assert np.array_equal(train_set["user"].values, gs["coo_u"]) and np.array_equal(train_set["item"].values, gs["coo_i"])
    model = MostPop(cfg)
    model.fit(train_set)
    out["ml_meta"] = np.array([cfg["user_num"], cfg["item_num"], cfg["topk"], cfg["seed"]], np.int64)
    out["ml_cnt"], out["ml_score"] = model.item_cnt_ref, model.item_score
    test_u, test_ucands = build_candidates_set(test_ur, train_ur, cfg)
    loader = get_dataloader(CandidatesDataset(test_ucands), batch_size=128, shuffle=False, num_workers=0)
    preds = model.rank(loader)
    out["ml_test_u"] = np.array(test_u, np.int32)
    out["ml_cands"] = np.stack([c[1] for c in test_ucands]).astype(np.int16)
    out["ml_rank"] = preds
    out["ml_full"] = model.full_rank(0)
    out["ml_predict"] = np.array([model.predict(0, i) for i in range(0, cfg["item_num"], 97)], np.float64)
    cfg["res_path"] = tempfile.mkdtemp() + "/"
    res = calc_ranking_results(test_ur, preds, test_u, cfg)
    out["ml_kpi"] = res.values[:, 1:].astype(np.float64)
    out["ml_kpi_ks"] = np.array([int(c) for c in res.columns[1:]], np.int32)
    print(res)


def main():
    rh.import_reference()
    _shims()
    out = {}
    gen_synthetic(out)
    gen_ml100k(out)
    path = os.path.join(GOLD, "mostpop.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}  ({os.path.getsize(path) / 1024:.1f} KiB)")


if __name__ == "__main__":
    main()
