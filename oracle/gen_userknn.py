"""Generates tests/golden/userknn.npz from the reference's own UserKNNCF (daisy/model/KNNCFRecommender.py:459-536), imported
through oracle/ref_harness.py with gen_itemknn.py's shims (the sparse ``.A`` property and a copying ``Tensor.numpy()``).

Synthetic data sets: gen_itemknn.py's d0 (star values, duplicate rows, users without rows), d1 (binary) and d2 (real values),
every configuration of gen_itemknn.configs() (maxk 600 >= U among them): w_sparse in full; for the configurations of SCORED
also rank on 30 candidates per user, pred_mat's entries for the first 24 users, full_rank of six users and predict.
ml-100k on config 1's split with assets/itemknn.yaml's values: a digest of w_sparse sorted per column, every 64th column in
full, rank on all test users with the reference's scores of the returned ids, full_rank, predict and the KPI table.

    python oracle/gen_userknn.py
"""
import os
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_harness as rh  # noqa: E402
from oracle.gen_itemknn import (COL_STRIDE, GOLD, SCORED, _datasets, _Loader, _shims, _w_sparse, configs, sha,  # noqa: E402
                                sorted_columns)


def gen_synthetic(out):
    import pandas as pd
    from daisy.model.KNNCFRecommender import UserKNNCF
    rng = np.random.default_rng(6)
    data = _datasets()
    cfgs = configs()
    for d, c in enumerate(data):
        df = pd.DataFrame({"user": c["u"].astype(np.int64), "item": c["i"].astype(np.int64), "rating": c["v"]})
        users = np.arange(c["U"], dtype=np.int64)
        cands = np.stack([rng.choice(c["I"], 30, replace=False) for _ in users]).astype(np.int64)
        out[f"d{d}_u"], out[f"d{d}_i"], out[f"d{d}_v"] = c["u"].astype(np.int16), c["i"].astype(np.int16), c["v"]
        out[f"d{d}_meta"] = np.array([c["U"], c["I"], 10], np.int64)
        out[f"d{d}_cands"] = cands.astype(np.int16)
        for k, (sim, nrm, sh, maxk) in enumerate(cfgs):
            cfg = rh.make_config("itemknn", user_num=c["U"], item_num=c["I"], topk=10, similarity=sim, normalize=nrm, shrink=sh,
                                 maxk=maxk)
            m = UserKNNCF(cfg)
            W = _w_sparse(lambda: m.fit(df))
            assert W.shape == (c["U"], c["U"]) and m.pred_mat.dtype == np.float64
            p = f"d{d}_c{k}"
            out[p + "_indptr"], out[p + "_indices"], out[p + "_data"] = W.indptr.astype(np.int32), W.indices.astype(np.int16), W.data
            if (sim, nrm, sh) in SCORED and maxk == 10:
                out[p + "_rank"] = m.rank(_Loader(users, cands)).astype(np.int16)
                out[p + "_scores"] = np.asarray(m.pred_mat[users[:24, None], cands[:24]].toarray(), np.float64)
                out[p + "_full"] = np.stack([m.full_rank(int(a)) for a in users[:6]]).astype(np.int16)
                out[p + "_predict"] = np.array([m.predict(int(a), int(b)) for a, b in zip(users, cands[:, 0])], np.float64)
    out["n_data"] = np.array(len(data))
    out["cfg_sim"] = np.array([c[0] for c in cfgs])
    out["cfg_normalize"] = np.array([c[1] for c in cfgs])
    out["cfg_shrink"] = np.array([c[2] for c in cfgs], np.int32)
    out["cfg_maxk"] = np.array([c[3] for c in cfgs], np.int32)


def gen_ml100k(out):
    from daisy.model.KNNCFRecommender import UserKNNCF
    from daisy.utils.dataset import CandidatesDataset, get_dataloader
    from daisy.utils.utils import build_candidates_set
    from daisy.utils.metrics import calc_ranking_results
    cfg = rh.make_config("itemknn")
    rh.seed_everything(cfg["seed"])
    art = rh.load_ml100k(cfg)
    train_set, test_ur, train_ur = art["train_set"], art["test_ur"], art["train_ur"]
    gs = np.load(os.path.join(GOLD, "ml100k_sampler.npz"))
    assert np.array_equal(train_set["user"].values, gs["coo_u"]) and np.array_equal(train_set["item"].values, gs["coo_i"])
    model = UserKNNCF(cfg)
    W = _w_sparse(lambda: model.fit(train_set))
    idx, val = sorted_columns(W)
    U = cfg["user_num"]
    out["ml_meta"] = np.array([U, cfg["item_num"], cfg["topk"], cfg["seed"], COL_STRIDE, cfg["maxk"], cfg["shrink"]], np.int64)
    out["ml_W_indptr"] = W.indptr.astype(np.int32)
    out["ml_W_val_sha"] = sha(W.indptr.astype(np.int64), val)
    out["ml_W_idx_sha"] = sha(idx)
    cols = np.arange(0, U, COL_STRIDE)
    Wc = W[:, cols]
    Wc.sort_indices()
    out["ml_Wc_indptr"], out["ml_Wc_indices"], out["ml_Wc_data"] = Wc.indptr.astype(np.int32), Wc.indices.astype(np.int16), Wc.data
    test_u, test_ucands = build_candidates_set(test_ur, train_ur, cfg)
    cands = np.stack([c[1] for c in test_ucands]).astype(np.int64)
    out["ml_cands_sha"] = sha(cands)
    loader = get_dataloader(CandidatesDataset(test_ucands), batch_size=128, shuffle=False, num_workers=0)
    preds = model.rank(loader)
    out["ml_test_u"] = np.array(test_u, np.int32)
    out["ml_rank"] = preds.astype(np.int16)
    P = model.pred_mat.tocsr()
    out["ml_rank_scores"] = np.stack([np.asarray(P[int(u), preds[k]].toarray()).ravel() for k, u in enumerate(test_u)])[:, :20]
    out["ml_full_u"] = np.array(test_u[:6], np.int32)
    out["ml_full"] = np.stack([model.full_rank(int(u)) for u in test_u[:6]]).astype(np.int16)
    pairs = np.array([[test_u[k], cands[k][-1 - k]] for k in range(8)], np.int64)
    out["ml_predict_pairs"] = pairs
    out["ml_predict"] = np.array([model.predict(int(u), int(i)) for u, i in pairs], np.float64)
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
    path = os.path.join(GOLD, "userknn.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}  ({os.path.getsize(path) / 1024:.1f} KiB)")


if __name__ == "__main__":
    main()
