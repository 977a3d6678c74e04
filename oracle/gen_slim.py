"""Generates tests/golden/slim.npz from the reference's own SLiM (daisy/model/SLiMRecommender.py), imported through
oracle/ref_harness.py.  Each column's ElasticNet result (coef_, dual_gap_, n_iter_) is captured by wrapping ``model.md.fit`` on
the instance; the reference source is not modified.  ``A_tilde`` is a lil_matrix whose ``.A`` current scipy no longer has:
gen_itemknn's shims (a ``.A`` property, ``Tensor.numpy()`` returning a copy) are applied for this process only.

Synthetic data sets, each fitted under CONFIGS with np.random.seed(SEED) before every fit, once with the reference's tol 1e-4 /
max_iter 100 and once on the same instance with ``md.tol`` = TIGHT_TOL and ``md.max_iter`` = TIGHT_ITER (every column must
converge):
  d0  star values with duplicate (u, i) rows, a cold item, users without rows      U 60,  I 40
  d1  binary                                                                       U 80,  I 36
  d2  positive real values                                                         U 100, I 34
  d3  real values including negatives                                              U 70,  I 32
Per (data set, configuration): coef_ of every column at both tolerances (sparse), dual_gap_, n_iter_; and for topk 5 and
topk 64 >= I: w_sparse, A_tilde rows of the first 8 users, rank on 30 candidates per user, full_rank of 4 users, predict on 8
pairs, and numpy's global state after fit.
ml-100k on config 1's split with assets/slim.yaml: w_sparse, the candidate digest, rank on all test users with the reference's
scores, full_rank of six users, predict on eight pairs, the calc_ranking_results table and numpy's state after fit.

    python oracle/gen_slim.py
"""
import os
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_harness as rh  # noqa: E402
from oracle.gen_itemknn import _Loader, _shims, sha  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
CONFIGS = ((1.0, 0.1), (0.05, 0.1), (0.01, 0.5), (0.1, 0.9))
TOPKS = (5, 64)
SEED = 2024
TIGHT_TOL, TIGHT_ITER = 1e-10, 100000


def datasets():
    rng = np.random.default_rng(41)
    out = []
    u, i = rng.integers(2, 60, 500), rng.integers(0, 39, 500)
    k = rng.integers(0, 500, 30)
    u, i = np.concatenate([u, u[k]]), np.concatenate([i, i[k]])
    out.append(dict(U=60, I=40, u=u, i=i, v=rng.integers(1, 6, len(u)).astype(np.float64)))
    u, i = rng.integers(0, 80, 700), rng.integers(0, 36, 700)
    out.append(dict(U=80, I=36, u=u, i=i, v=np.ones(700)))
    u, i = rng.integers(0, 100, 900), rng.integers(0, 34, 900)
    out.append(dict(U=100, I=34, u=u, i=i, v=rng.random(900) * 3.0 + 0.01))
    u, i = rng.integers(0, 70, 600), rng.integers(0, 32, 600)
    out.append(dict(U=70, I=32, u=u, i=i, v=rng.integers(-2, 5, 600).astype(np.float64)))
    return out


def _capture(model):
    """Wrap model.md.fit to record each column's coef_, dual_gap_, n_iter_."""
    rec = []
    md = model.md
    fit = type(md).fit

    def wrapped(X, y, *a, **k):
        r = fit(md, X, y, *a, **k)
        rec.append((np.array(md.coef_, np.float64).ravel(), float(md.dual_gap_), int(np.max(md.n_iter_))))
        return r

    md.fit = wrapped
    return rec


def _fit(model, df, tol=None, max_iter=None):
    if tol is not None:
        model.md.tol, model.md.max_iter = tol, max_iter
    rec = _capture(model)
    np.random.seed(SEED)
    model.fit(df, verbose=False)
    coef = np.stack([r[0] for r in rec], 1)               # [I, I], column j item j's coefficients
    return coef, np.array([r[1] for r in rec]), np.array([r[2] for r in rec], np.int32)


def _state_sha():
    st = np.random.get_state()
    return sha(np.asarray(st[1], np.uint32), np.array([st[2], st[3]], np.int64))


def _put_sparse(out, p, M):
    import scipy.sparse as sp
    C = sp.csc_matrix(M)
    C.sort_indices()
    out[p + "_indptr"], out[p + "_indices"], out[p + "_data"] = C.indptr.astype(np.int32), C.indices.astype(np.int16), C.data


def gen_synthetic(out):
    import pandas as pd
    from daisy.model.SLiMRecommender import SLiM
    rng = np.random.default_rng(6)
    for d, c in enumerate(datasets()):
        df = pd.DataFrame({"user": c["u"].astype(np.int64), "item": c["i"].astype(np.int64), "rating": c["v"]})
        users = np.arange(c["U"], dtype=np.int64)
        cands = np.stack([rng.choice(c["I"], 30, replace=False) for _ in users]).astype(np.int64)
        out[f"d{d}_u"], out[f"d{d}_i"], out[f"d{d}_v"] = c["u"].astype(np.int16), c["i"].astype(np.int16), c["v"]
        out[f"d{d}_meta"] = np.array([c["U"], c["I"]], np.int64)
        out[f"d{d}_cands"] = cands.astype(np.int16)
        for k, (alpha, elastic) in enumerate(CONFIGS):
            for t, topk in enumerate(TOPKS):
                p = f"d{d}_c{k}_t{t}"
                cfg = rh.make_config("slim", user_num=c["U"], item_num=c["I"], topk=topk, alpha=alpha, elastic=elastic)
                m = SLiM(cfg)
                coef, gaps, iters = _fit(m, df)
                out[p + "_rng"] = _state_sha()
                W = m.w_sparse.tocsr()
                W.sort_indices()
                out[p + "_W_indptr"], out[p + "_W_indices"], out[p + "_W_data"] = W.indptr.astype(np.int32), W.indices.astype(np.int16), W.data
                A = m.A_tilde.tocsr()
                out[p + "_A"] = np.asarray(A[:8].toarray(), np.float64)
                out[p + "_rank"] = m.rank(_Loader(users, cands)).astype(np.int16)
                out[p + "_full"] = np.stack([m.full_rank(int(a)) for a in users[:4]]).astype(np.int16)
                out[p + "_predict"] = np.array([m.predict(int(a), int(b)) for a, b in zip(users[:8], cands[:8, 0])], np.float64)
                if t == 0:                                 # the fit does not depend on topk
                    q = f"d{d}_c{k}"
                    _put_sparse(out, q + "_coef", coef)
                    out[q + "_gap"], out[q + "_iter"] = gaps, iters
                    coef2, gaps2, iters2 = _fit(m, df, TIGHT_TOL, TIGHT_ITER)
                    assert np.all(iters2 < TIGHT_ITER), "a column did not converge at the tight tolerance"
                    _put_sparse(out, q + "_coeft", coef2)
                    out[q + "_gapt"], out[q + "_itert"] = gaps2, iters2
    out["n_data"] = np.array(len(datasets()))
    out["configs"] = np.array(CONFIGS, np.float64)
    out["topks"] = np.array(TOPKS, np.int32)
    out["seed"] = np.array(SEED)
    out["tight"] = np.array([TIGHT_TOL, TIGHT_ITER], np.float64)


def gen_ml100k(out):
    from daisy.model.SLiMRecommender import SLiM
    from daisy.utils.dataset import CandidatesDataset, get_dataloader
    from daisy.utils.utils import build_candidates_set
    from daisy.utils.metrics import calc_ranking_results
    cfg = rh.make_config("slim")
    rh.seed_everything(cfg["seed"])
    art = rh.load_ml100k(cfg)
    train_set, test_ur, train_ur = art["train_set"], art["test_ur"], art["train_ur"]
    gs = np.load(os.path.join(GOLD, "ml100k_sampler.npz"))         # config 1's split: the rows of ml100k_sampler.npz
    assert np.array_equal(train_set["user"].values, gs["coo_u"]) and np.array_equal(train_set["item"].values, gs["coo_i"])
    out["ml_rng_before"] = _state_sha()
    model = SLiM(cfg)
    model.fit(train_set, verbose=False)
    out["ml_rng"] = _state_sha()
    W = model.w_sparse.tocsr()
    W.sort_indices()
    out["ml_W_indptr"], out["ml_W_indices"], out["ml_W_data"] = W.indptr.astype(np.int32), W.indices.astype(np.int16), W.data
    out["ml_meta"] = np.array([cfg["user_num"], cfg["item_num"], cfg["topk"], cfg["seed"]], np.int64)
    out["ml_alpha_elastic"] = np.array([cfg["alpha"], cfg["elastic"]], np.float64)
    test_u, test_ucands = build_candidates_set(test_ur, train_ur, cfg)
    cands = np.stack([c[1] for c in test_ucands]).astype(np.int64)
    out["ml_cands_sha"] = sha(cands)
    loader = get_dataloader(CandidatesDataset(test_ucands), batch_size=128, shuffle=False, num_workers=0)
    preds = model.rank(loader)
    out["ml_test_u"] = np.array(test_u, np.int32)
    out["ml_rank"] = preds.astype(np.int16)
    A = model.A_tilde.tocsr()
    out["ml_rank_scores"] = np.stack([np.asarray(A[int(u), preds[k]].toarray()).ravel() for k, u in enumerate(test_u)])
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
    path = os.path.join(GOLD, "slim.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}  ({os.path.getsize(path) / 1024:.1f} KiB)")


if __name__ == "__main__":
    main()
