"""EASE on the GPU path (csrc/ease.cu, daisyrec_b200/model/EASERecommender.py) against host references: scipy / numpy for X,
the Gram and the inverse, and the numpy restatement in oracle/ease_oracle.py for the scoring."""
import logging

import numpy as np
import pandas as pd
import pytest
import torch

from oracle import ease_oracle as eo

pytestmark = pytest.mark.gpu


def _coo(U, I, nnz, seed, values='binary', dups=0):
    rng = np.random.default_rng(seed)
    u = rng.integers(U, size=nnz)
    i = rng.integers(I, size=nnz)
    if dups:                                               # repeat some pairs, with other values
        k = rng.integers(nnz, size=dups)
        u, i = np.concatenate([u, u[k]]), np.concatenate([i, i[k]])
    n = len(u)
    if values == 'binary':
        v = np.ones(n)
    elif values == 'stars':
        v = rng.integers(1, 6, size=n).astype(np.float64)
    elif values == 'half':
        v = rng.integers(1, 11, size=n) * 0.5
    else:
        v = rng.random(n) * 3.0 + 0.01
    return u, i, v


def _X(u, i, v, U, I):
    from daisyrec_b200 import ops
    d = lambda a, t: torch.from_numpy(np.ascontiguousarray(a, t)).cuda()
    return ops.ease_csr(d(u, np.int32), d(i, np.int32), d(v, np.float64), U, I)


def _host_x(X):
    import scipy.sparse as sp
    return sp.csr_matrix((X.val.cpu().numpy(), X.col.cpu().numpy(), X.row_ptr.cpu().numpy()), shape=(X.user_num, X.item_num))


def _gram(X, reg, scale=None):
    from daisyrec_b200 import ops
    ws = ops.ease_workspace(X, scale)
    return ops.ease_gram(X, reg, ws, scale=scale), ws


# ------------------------------------------------------------------ X
@pytest.mark.parametrize("values,dups,scale", [("binary", 0, 0), ("stars", 300, 0), ("half", 300, 1), ("real", 300, -1)])
def test_csr_values_and_scale(values, dups, scale):
    U, I = 500, 333
    u, i, v = _coo(U, I, 6000, 1, values, dups)
    X = _X(u, i, v, U, I)
    ref = eo.interaction_matrix(u, i, v, U, I)
    ref.sort_indices()
    got = _host_x(X)
    assert np.array_equal(got.indptr, ref.indptr) and np.array_equal(got.indices, ref.indices)
    assert np.array_equal(got.data, ref.data)                                  # fp64 sums rounded once to fp32
    assert X.scale == eo.exact_scale(ref) == scale


def test_scale_refuses_overflowing_columns():
    # one column of 133 200 users: 133 200 * 127^2 = 2.148e9 >= 2^31 (refused), 133 200 * 126^2 = 2.115e9 (exact)
    U, I = 133200, 3
    u = np.arange(U)
    i = np.zeros(U, np.int64)
    X = _X(u, i, np.full(U, 127.0), U, I)
    assert X.scale == -1
    X = _X(u, i, np.full(U, 126.0), U, I)
    assert X.scale == 0


# ------------------------------------------------------------------ Gram
@pytest.mark.parametrize("U,I,values,dups", [(300, 1, "binary", 0), (1000, 129, "binary", 500), (977, 300, "half", 400),
                                             (70000, 9000, "binary", 0), (2000, 515, "stars", 1000)])
def test_gram_exact_bitwise(U, I, values, dups):
    nnz = min(U * I // 3, 60 * U)
    u, i, v = _coo(U, I, nnz, 7, values, dups)
    u[u == U - 2] = U - 1                                 # a user without rows
    if I > 1:
        i[i == I - 1] = 0                                 # a cold item
    X = _X(u, i, v, U, I)
    assert X.scale >= 0
    G, _ = _gram(X, 200.0)
    h = _host_x(X)
    q = (h.astype(np.float64) * 2.0 ** X.scale).astype(np.int64)
    ref = (q.T @ q).toarray().astype(np.float64) * 2.0 ** (-2 * X.scale) + 200.0 * np.eye(I)
    assert np.array_equal(G.cpu().numpy(), ref)
    if I == 9000:                                        # more than one user chunk at this shape
        from daisyrec_b200 import _lib as L
        assert L.lib().drb_ease_workspace_bytes(U, I, 0) < U * 9088


@pytest.mark.parametrize("U,I", [(500, 1), (1500, 333), (4000, 1000)])
def test_gram_general_path(U, I):
    u, i, v = _coo(U, I, 20 * U, 3, "real", 200)
    X = _X(u, i, v, U, I)
    assert X.scale == -1
    G, _ = _gram(X, 5.0)
    h = _host_x(X).astype(np.float64)
    ref = (h.T @ h).toarray() + 5.0 * np.eye(I)
    bound = (abs(h).T @ abs(h)).toarray() + 5.0 * np.eye(I)
    assert np.all(np.abs(G.cpu().numpy() - ref) <= 1e-13 * bound)
    # the binary data of the exact path, forced through fp64 DMMA, gives the same integers
    X1 = _X(u, i, np.ones(len(u)), U, I)
    G0, _ = _gram(X1, 1.0)
    G1, _ = _gram(X1, 1.0, scale=-1)
    assert torch.equal(G0, G1)


# ------------------------------------------------------------------ inverse
def _fit_dense(X, reg):
    from daisyrec_b200 import ops
    G, ws = _gram(X, reg)
    G0 = G.clone()
    ops.ease_inverse(G, ws)
    return G0, G, ws


@pytest.mark.parametrize("n", [1, 63, 64, 65, 1152, 3000])
def test_inverse(n):
    from daisyrec_b200 import ops
    U = max(50, 3 * n)
    u, i, v = _coo(U, n, 12 * U, n, "binary")
    X = _X(u, i, v, U, n)
    G0, P, ws = _fit_dense(X, 20.0)
    res = (G0 @ P - torch.eye(n, dtype=torch.float64, device='cuda')).abs().max().item()
    assert res <= 1e-10, res
    Ph = P.cpu().numpy()
    ref = np.linalg.inv(G0.cpu().numpy())
    assert np.abs(Ph - ref).max() <= 1e-11 * np.abs(ref).max()
    assert np.array_equal(Ph, Ph.T)
    B = ops.ease_weights(P.clone(), ws).cpu().numpy()
    assert np.all(np.diag(B) == 0)
    want = -Ph / np.diag(Ph)
    np.fill_diagonal(want, 0.)
    assert np.array_equal(B, want)


def test_inverse_ml20m_shape_and_reproducible():
    from daisyrec_b200 import ops
    from daisyrec_b200.utils import synthetic
    U, I, nnz = 138493, 26744, 20_000_263
    d = synthetic.make_interactions(U, I, nnz, device="cuda")
    n = d["coo_u"].numel()
    X = ops.ease_csr(d["coo_u"], d["coo_i"], torch.ones(n, dtype=torch.float64, device="cuda"), U, I)
    assert X.scale == 0
    ws = ops.ease_workspace(X)
    G = ops.ease_gram(X, 500.0, ws)
    G0 = G.clone()
    ops.ease_inverse(G, ws)
    R = G0 @ G
    R.diagonal().sub_(1.0)
    res = R.abs().max().item()
    del R
    assert res <= 1e-10, res
    B1 = ops.ease_weights(G, ws)
    del G0
    G2 = ops.ease_gram(X, 500.0, ws)
    ops.ease_weights(ops.ease_inverse(G2, ws), ws)
    assert torch.equal(B1, G2)


def test_not_positive_definite():
    from daisyrec_b200 import ops
    G = torch.eye(70, dtype=torch.float64, device='cuda')
    G[40, 40] = -1.0
    ws = torch.empty(1 << 22, dtype=torch.uint8, device='cuda')
    with pytest.raises(np.linalg.LinAlgError):
        ops.ease_inverse(G, ws)


# ------------------------------------------------------------------ scoring
def _fitted(U=600, I=700, seed=5, values="binary"):
    from daisyrec_b200 import ops
    u, i, v = _coo(U, I, 15 * U, seed, values, 100)
    u[u < 10] = 10                                        # users 0..9 have no rows
    X = _X(u, i, v, U, I)
    G0, P, ws = _fit_dense(X, 50.0)
    B = ops.ease_weights(P, ws)
    return X, B


def _gap_ok(s, k):
    """rows whose top-(k+1) scores are separated by >= 1e-10 relative (ids are then exact)."""
    srt = -np.sort(-s, axis=1)[:, :k + 1]
    gaps = np.abs(np.diff(srt, axis=1)) / np.maximum(np.abs(srt[:, :-1]), 1e-300)
    return np.all(gaps >= 1e-10, axis=1)


def test_rank_full_rank_predict_against_oracle():
    from daisyrec_b200 import ops
    X, B = _fitted()
    Xh, Bh = _host_x(X), B.cpu().numpy()
    rng = np.random.default_rng(0)
    users = rng.integers(X.user_num, size=300)
    users[:5] = np.arange(5)                             # no train rows: all scores 0
    cands = np.stack([rng.choice(X.item_num, 120, replace=False) for _ in range(300)])
    ids, sc = ops.ease_rank(B, X, torch.from_numpy(users).cuda(), torch.from_numpy(cands).cuda(), 50, scores=True)
    want_ids, want_sc = eo.rank(Xh, Bh, users, cands, 50)
    sc = sc.cpu().numpy()
    Xa, Ba = abs(Xh), np.abs(Bh)                          # scores are sums that cancel: relative to sum |x_ui B_ci|
    assert np.all(np.abs(sc - want_sc) <= 1e-12 * eo.rank_scores(Xa, Ba, users, cands))
    ok = _gap_ok(want_sc, 50)
    assert ok.sum() > 250
    assert np.array_equal(ids.cpu().numpy()[ok], want_ids[ok])
    assert np.array_equal(ids.cpu().numpy()[:5], cands[:5, :50])        # all-zero rows: the first positions
    # full_rank and predict use x B, rank uses x B^T
    fr, fsc = ops.ease_full_rank(B, X, torch.from_numpy(users[:40]).cuda(), 50, scores=True)
    want_fr, want_fsc = eo.full_rank(Xh, Bh, users[:40], 50)
    fsc = fsc.cpu().numpy()
    assert np.all(np.abs(fsc - want_fsc) <= 1e-12 * eo.user_scores(Xa, Ba, users[:40]))
    ok = _gap_ok(want_fsc, 50)
    assert np.array_equal(fr.cpu().numpy()[ok], want_fr[ok])
    assert np.array_equal(fr.cpu().numpy()[:5], np.tile(np.arange(50), (5, 1)))
    pi = cands[:, 0]
    pr = ops.ease_predict(B, X, torch.from_numpy(users).cuda(), torch.from_numpy(pi).cuda()).cpu().numpy()
    want_p = np.array([eo.predict(Xh, Bh, int(a), int(b)) for a, b in zip(users, pi)])
    assert np.all(np.abs(pr - want_p) <= 1e-12 * np.array([eo.predict(Xa, Ba, int(a), int(b)) for a, b in zip(users, pi)]))
    # the quirk: rank's scores are x B^T, not x B
    xb = eo.user_scores(Xh, Bh, users)
    alt = np.take_along_axis(xb, cands, 1)
    assert not np.allclose(alt[5:], sc[5:])


def _config(**kw):
    cfg = dict(gpu='0', reg=50.0, topk=50, user_num=600, item_num=700, UID_NAME='user', IID_NAME='item', INTER_NAME='rating',
               logger=logging.getLogger('t'))
    cfg.update(kw)
    return cfg


class _Loader:
    def __init__(self, users, cands, bs=128):
        self.users, self.cands, self.bs = users, cands, bs

    def __iter__(self):
        for s in range(0, len(self.users), self.bs):
            yield torch.from_numpy(self.users[s:s + self.bs]), torch.from_numpy(self.cands[s:s + self.bs])


def test_class_surface():
    from daisyrec_b200.model import EASE
    U, I = 600, 700
    u, i, v = _coo(U, I, 9000, 11, "stars", 200)
    df = pd.DataFrame({'user': u, 'item': i, 'rating': v})
    m = EASE(_config())
    m.fit(df)
    Xr, Gr, Pr, Br = eo.fit(u, i, v, U, I, 50.0)
    assert m.item_similarity.dtype == torch.float64 and m.item_similarity.shape == (I, I)
    Bh = m.item_similarity.cpu().numpy()
    assert np.abs(Bh - Br).max() <= 1e-10 * np.abs(Br).max()
    Xr.sort_indices()
    xm = m.interaction_matrix
    assert xm.dtype == np.float32 and (xm != Xr).nnz == 0
    rng = np.random.default_rng(1)
    users = rng.integers(U, size=200)
    cands = np.stack([rng.choice(I, 100, replace=False) for _ in range(200)])
    got = m.rank(_Loader(users, cands))
    assert got.dtype == np.int64 and got.shape == (200, 50)
    want, s = eo.rank(Xr, Bh, users, cands, 50)
    ok = _gap_ok(s, 50)
    assert np.array_equal(got[ok], want[ok])
    fr = m.full_rank(3)
    assert fr.dtype == np.int64 and fr.shape == (1, 50)
    p = m.predict(3, 4)
    assert isinstance(p, np.float64)
    assert abs(p - eo.predict(Xr, Bh, 3, 4)) <= 1e-9 * eo.predict(abs(Xr), np.abs(Bh), 3, 4)
    # refusals
    with pytest.raises(IndexError):
        m.predict(U, 0)
    with pytest.raises(IndexError):
        m.predict(0, I)
    with pytest.raises(IndexError):
        m.full_rank(-1)
    with pytest.raises(IndexError):
        m.rank(_Loader(users, np.where(cands == cands[0, 0], I, cands)))
    bad = df.copy()
    bad.loc[0, 'item'] = I
    with pytest.raises(ValueError):
        EASE(_config()).fit(bad)
    bad = df.copy()
    bad.loc[0, 'user'] = -1
    with pytest.raises(ValueError):
        EASE(_config()).fit(bad)
    for reg in (0.0, -1.0):
        with pytest.raises(NotImplementedError, match='positive definite'):
            EASE(_config(reg=reg)).fit(df)


# ------------------------------------------------------------------ against the reference's runs (tests/golden/ease.npz)
def test_synthetic_cases_vs_reference():
    from daisyrec_b200.model import EASE
    from conftest import golden
    g = golden("ease")
    for k in range(int(g["n_synthetic"])):
        U, I, topk = (int(v) for v in g[f"s{k}_meta"])
        u, i, v = g[f"s{k}_u"], g[f"s{k}_i"], g[f"s{k}_v"]
        m = EASE(_config(user_num=U, item_num=I, topk=topk, reg=float(g[f"s{k}_reg"])))
        m.fit(pd.DataFrame({'user': u.astype(np.int64), 'item': i.astype(np.int64), 'rating': v}))
        Xh = m.interaction_matrix
        exact = eo.exact_scale(Xh) >= 0
        B, want_B = m.item_similarity.cpu().numpy(), g[f"s{k}_B"]
        # real weights: the reference's Gram is an fp32 sparse product that rounds
        assert np.abs(B - want_B).max() <= (1e-10 if exact else 1e-6) * np.abs(want_B).max(), k
        assert np.all(np.diag(B) == 0)
        users = np.arange(U)
        cands = g[f"s{k}_cands"].astype(np.int64)
        got = m.rank(_Loader(users, cands, bs=16))
        ok = _gap_ok(eo.rank_scores(Xh, want_B, users, cands), topk)
        if not exact:
            srt = -np.sort(-eo.rank_scores(Xh, want_B, users, cands), axis=1)[:, :topk + 1]
            ok &= np.all(np.abs(np.diff(srt, axis=1)) >= 1e-5 * np.abs(srt).max(), axis=1)
        zero = np.diff(Xh.indptr)[users] == 0
        assert np.array_equal(got[ok | zero], g[f"s{k}_rank"][ok | zero]), k
        assert (ok | zero).sum() >= 0.8 * U, k
        full = np.concatenate([m.full_rank(int(a)) for a in users[:6]])
        assert np.array_equal(full[zero[:6] | exact], g[f"s{k}_full"][zero[:6] | exact]), k
        pred = np.array([m.predict(int(a), int(b)) for a, b in zip(users, cands[:, 0])])
        bound = np.array([eo.predict(abs(Xh), np.abs(want_B), int(a), int(b)) for a, b in zip(users, cands[:, 0])])
        assert np.all(np.abs(pred - g[f"s{k}_predict"]) <= (1e-9 if exact else 1e-5) * bound + 1e-300), k


def test_ml100k_driver_sequence():
    """test.py's ease branch on config 1's ml-100k split through the drop-in classes: EASE(config).fit(train_set) ->
    build_candidates_set -> rank -> calc_ranking_results, and full_rank / predict, against the reference's run."""
    import hashlib
    import tempfile
    from conftest import golden
    from daisyrec_b200 import ops
    from daisyrec_b200.model import EASE
    from daisyrec_b200.utils.dataset import CandidatesDataset, get_dataloader
    from daisyrec_b200.utils.metrics import calc_ranking_results
    from daisyrec_b200.utils.utils import get_ur, build_candidates_set
    g, gs, gr = golden("ease"), golden("ml100k_sampler"), golden("ml100k_rank")
    U, I, topk, seed, stride = (int(v) for v in g["ml_meta"])
    reg = float(g["ml_reg"])
    train_set = pd.DataFrame({'user': gs["coo_u"].astype(np.int64), 'item': gs["coo_i"].astype(np.int64), 'rating': 1.0})
    off = np.concatenate([[0], np.cumsum(gr["gt_len"])])
    # the reference's test sets in their own iteration order (candidates end with list(test_ur[u]))
    test_ur = {int(u): gr["gt_flat"][off[k]:off[k + 1]].tolist() for k, u in enumerate(gr["test_u"])}
    cfg = _config(user_num=U, item_num=I, topk=topk, reg=reg, cand_num=1000, seed=seed)
    np.random.seed(seed); torch.manual_seed(seed)
    train_ur = get_ur(train_set)
    model = EASE(cfg)
    model.fit(train_set)
    X = model.interaction_matrix
    h = hashlib.sha256()
    for a in (X.indptr.astype(np.int64), X.indices.astype(np.int32), X.data.astype(np.float32)):
        h.update(np.ascontiguousarray(a).tobytes())
    assert h.digest() == g["ml_X_sha"].tobytes()
    B = model.item_similarity.cpu().numpy()
    rows = np.concatenate([B[:2], B[::stride]])
    assert np.abs(rows - g["ml_B_rows"]).max() <= 1e-10 * np.abs(g["ml_B_rows"]).max()
    assert np.abs(B.sum(0) - g["ml_B_colsum"]).max() <= 1e-10 * np.abs(B).sum(0).max()
    # P of the same fit, stopped before B
    d = lambda a, t: torch.from_numpy(np.ascontiguousarray(a, t)).cuda()
    Xd = ops.ease_csr(d(gs["coo_u"], np.int32), d(gs["coo_i"], np.int32), d(np.ones(len(gs["coo_u"])), np.float64), U, I)
    ws = ops.ease_workspace(Xd)
    P = ops.ease_inverse(ops.ease_gram(Xd, reg, ws), ws)
    assert np.allclose(P.diagonal().cpu().numpy(), g["ml_P_diag"], rtol=1e-11, atol=0)
    # test.py:112-131
    test_u, test_ucands = build_candidates_set(test_ur, train_ur, cfg)
    cands = np.stack([np.asarray(c[1], np.int64) for c in test_ucands])
    assert hashlib.sha256(cands.tobytes()).digest() == g["ml_cands_sha"].tobytes()
    preds = model.rank(get_dataloader(CandidatesDataset(test_ucands), batch_size=128, shuffle=False, num_workers=0))
    assert preds.dtype == np.int64 and preds.shape == g["ml_rank"].shape
    assert np.array_equal(preds, g["ml_rank"])                                 # all 304 rows
    for k, u in enumerate(g["ml_full_u"]):
        f = model.full_rank(int(u))
        assert f.dtype == np.int64 and f.shape == (1, topk)
        assert np.array_equal(f[0], g["ml_full"][k])
    for (u, i), want in zip(g["ml_predict_pairs"], g["ml_predict"]):
        p = model.predict(int(u), int(i))
        assert isinstance(p, np.float64) and abs(p - want) <= 1e-9 * abs(want)
    kcfg = dict(logger=logging.getLogger('t'), res_path=tempfile.mkdtemp() + '/', metrics=["recall", "mrr", "ndcg", "hit", "precision"],
                item_num=I, topk=topk)
    res = calc_ranking_results(test_ur, preds, test_u, kcfg)
    assert [int(c) for c in res.columns[1:]] == g["ml_kpi_ks"].tolist()
    np.testing.assert_allclose(res.values[:, 1:].astype(np.float64), g["ml_kpi"], rtol=1e-12, atol=1e-12)
