"""Generates tests/golden/itemknn.npz from the reference's own ItemKNNCF (daisy/model/KNNCFRecommender.py), imported through
oracle/ref_harness.py.  The reference's rank / full_rank read ``lil_matrix[...].A``, an attribute current scipy no longer has:
the sparse classes get an ``A`` property returning ``toarray()`` here, for this process only.  scipy's fancy indexing also
re-flags its index arrays writeable, which numpy refuses for arrays that view a tensor's memory: ``Tensor.numpy()`` returns a
copy here.

Synthetic data sets (w_sparse in full for every configuration below; rank on 30 candidates per user, pred_mat's entries for the first 24 users, full_rank
and predict for the configurations of SCORED):
  d0  star values with duplicate (u, i) rows, a cold item, users without rows      U 60,  I 45
  d1  binary                                                                       U 80,  I 65
  d2  real-valued weights                                                          U 150, I 70
Configurations: cosine / asymmetric / adjusted / pearson x normalize {True, False} x shrink {0, 100}, jaccard / tanimoto / dice /
tversky x shrink {0, 100}, all with maxk 10, and cosine with maxk 600 >= I.
ml-100k on config 1's split with assets/itemknn.yaml (cosine, shrink 100, maxk 40): a digest of w_sparse sorted per column by
(value descending, id ascending), every 64th column in full, rank on all test users with the reference's scores of the returned
ids, full_rank of six users, predict on eight pairs, and the calc_ranking_results table.

    python oracle/gen_itemknn.py
"""
import hashlib
import os
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_harness as rh  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
COL_STRIDE = 64
SCORED = (("cosine", True, 100), ("pearson", True, 0), ("jaccard", False, 0), ("cosine", False, 100))


def _shims():
    import scipy.sparse as sp
    import torch
    to_numpy = torch.Tensor.numpy
    torch.Tensor.numpy = lambda self, *a, **k: np.array(to_numpy(self, *a, **k))
    for name in dir(sp):
        cls = getattr(sp, name)
        if isinstance(cls, type) and hasattr(cls, "toarray") and not hasattr(cls, "A"):
            cls.A = property(lambda self: self.toarray())


def sha(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return np.frombuffer(h.digest(), np.uint8)


def configs():
    out = []
    for sim in ("cosine", "asymmetric", "adjusted", "pearson"):
        out += [(sim, nrm, sh, 10) for nrm in (True, False) for sh in (0, 100)]
    for sim in ("jaccard", "tanimoto", "dice", "tversky"):
        out += [(sim, False, sh, 10) for sh in (0, 100)]
    return out + [("cosine", True, 100, 600)]


def _datasets():
    rng = np.random.default_rng(33)
    out = []
    u = rng.integers(2, 60, 700)
    i = rng.integers(0, 44, 700)
    k = rng.integers(0, 700, 40)
    u, i = np.concatenate([u, u[k]]), np.concatenate([i, i[k]])
    out.append(dict(U=60, I=45, u=u, i=i, v=rng.integers(1, 6, len(u)).astype(np.float64)))
    u, i = rng.integers(0, 80, 900), rng.integers(0, 65, 900)
    out.append(dict(U=80, I=65, u=u, i=i, v=np.ones(900)))
    u, i = rng.integers(0, 150, 2000), rng.integers(0, 70, 2000)
    out.append(dict(U=150, I=70, u=u, i=i, v=rng.random(2000) * 3.0 + 0.01))
    return out


class _Loader:
    """(us, cands_ids) batches, as the reference's rank iterates its test loader."""

    def __init__(self, users, cands, bs=16):
        self.users, self.cands, self.bs = users, cands, bs

    def __iter__(self):
        import torch
        for s in range(0, len(self.users), self.bs):
            yield torch.from_numpy(self.users[s:s + self.bs]), torch.from_numpy(self.cands[s:s + self.bs])


def _w_sparse(fit):
    """Run fit and catch the csc w_sparse it builds (the model keeps only pred_mat)."""
    import scipy.sparse as sp
    seen = []
    tocsc = sp.csr_matrix.tocsc

    def rec(self, *a, **k):
        r = tocsc(self, *a, **k)
        seen.append(r)
        return r

    sp.csr_matrix.tocsc = rec
    try:
        fit()
    finally:
        sp.csr_matrix.tocsc = tocsc
    W = [w for w in seen if w.shape[0] == w.shape[1] and w.dtype == np.float32][-1]
    W.sort_indices()
    return W


def gen_synthetic(out):
    import pandas as pd
    from daisy.model.KNNCFRecommender import ItemKNNCF
    rng = np.random.default_rng(5)
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
            m = ItemKNNCF(cfg)
            W = _w_sparse(lambda: m.fit(df))
            assert m.pred_mat.dtype == np.float64 and W.dtype == np.float32
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
    out["dtypes"] = np.array(["float32", "float64"])            # w_sparse, pred_mat


def sorted_columns(W):
    """(indices, data) of a csc matrix with every column ordered by (value descending, id ascending)."""
    idx, val = W.indices.astype(np.int32).copy(), W.data.copy()
    for c in range(W.shape[1]):
        s = slice(W.indptr[c], W.indptr[c + 1])
        o = np.lexsort((idx[s], -val[s]))
        idx[s], val[s] = idx[s][o], val[s][o]
    return idx, val


def gen_ml100k(out):
    from daisy.model.KNNCFRecommender import ItemKNNCF
    from daisy.utils.dataset import CandidatesDataset, get_dataloader
    from daisy.utils.utils import build_candidates_set
    from daisy.utils.metrics import calc_ranking_results
    cfg = rh.make_config("itemknn")
    rh.seed_everything(cfg["seed"])
    art = rh.load_ml100k(cfg)
    train_set, test_ur, train_ur = art["train_set"], art["test_ur"], art["train_ur"]
    gs = np.load(os.path.join(GOLD, "ml100k_sampler.npz"))         # config 1's split: the rows of ml100k_sampler.npz
    assert np.array_equal(train_set["user"].values, gs["coo_u"]) and np.array_equal(train_set["item"].values, gs["coo_i"])
    assert np.all(train_set["rating"].values == 1.0)
    model = ItemKNNCF(cfg)
    W = _w_sparse(lambda: model.fit(train_set))
    idx, val = sorted_columns(W)
    I = cfg["item_num"]
    out["ml_meta"] = np.array([cfg["user_num"], I, cfg["topk"], cfg["seed"], COL_STRIDE, cfg["maxk"], cfg["shrink"]], np.int64)
    out["ml_W_indptr"] = W.indptr.astype(np.int32)
    out["ml_W_val_sha"] = sha(W.indptr.astype(np.int64), val)
    out["ml_W_idx_sha"] = sha(idx)
    cols = np.arange(0, I, COL_STRIDE)
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
    nrow = np.bincount(gs["coo_u"], minlength=cfg["user_num"])
    warm = [u for u in test_u if nrow[u] > 0][:4]
    cold = [u for u in range(cfg["user_num"]) if nrow[u] == 0][:2]
    out["ml_full_u"] = np.array(warm + cold, np.int32)
    out["ml_full"] = np.stack([model.full_rank(int(u)) for u in warm + cold]).astype(np.int16)
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
    path = os.path.join(GOLD, "itemknn.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}  ({os.path.getsize(path) / 1024:.1f} KiB)")


if __name__ == "__main__":
    main()
