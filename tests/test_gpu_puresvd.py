"""PureSVD on the GPU path (csrc/puresvd.cu, daisyrec_b200/model/PureSVDRecommender.py) against scipy / numpy for the kernels,
the numpy restatement in oracle/puresvd_oracle.py, and the reference's own runs in tests/golden/puresvd.npz."""
import hashlib
import logging
import tempfile

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp
import torch

from conftest import golden
from oracle import puresvd_oracle as po
from test_puresvd_cpu import check_factors

pytestmark = pytest.mark.gpu


def _d(a, t):
    return torch.from_numpy(np.ascontiguousarray(a, t)).cuda()


def _coo(U, I, nnz, seed, dups=0, real=False):
    rng = np.random.default_rng(seed)
    u, i = rng.integers(U, size=nnz), rng.integers(I, size=nnz)
    if dups:
        k = rng.integers(nnz, size=dups)
        u, i = np.concatenate([u, u[k]]), np.concatenate([i, i[k]])
    v = rng.random(len(u)) * 3.0 + 0.01 if real else rng.integers(1, 6, len(u)).astype(np.float64)
    return u, i, v


def _X(u, i, v, U, I):
    from daisyrec_b200 import ops
    return ops.puresvd_csr(_d(u, np.int32), _d(i, np.int32), _d(v, np.float64), U, I)


def _config(**kw):
    cfg = dict(gpu='0', factors=10, topk=10, user_num=100, item_num=80, logger=logging.getLogger('t'))
    cfg.update(kw)
    return cfg


class _Loader:
    def __init__(self, users, cands, bs=128):
        self.users, self.cands, self.bs = users, cands, bs

    def __iter__(self):
        for s in range(0, len(self.users), self.bs):
            yield torch.from_numpy(self.users[s:s + self.bs]), torch.from_numpy(self.cands[s:s + self.bs])


# ------------------------------------------------------------------ X
def test_csr_matches_scipy():
    U, I = 700, 450
    u, i, v = _coo(U, I, 9000, 1, dups=800, real=True)
    u[u == 5] = 6                                                # a user without rows
    X = _X(u, i, v, U, I)
    ref = po.interaction_matrix(u, i, v, U, I)
    assert np.array_equal(X.row_ptr.cpu().numpy(), ref.indptr) and np.array_equal(X.col.cpu().numpy(), ref.indices)
    sums = {}
    for a, b, x in zip(u.tolist(), i.tolist(), v.tolist()):      # fp64 sums in row order
        sums[(a, b)] = sums.get((a, b), 0.0) + x
    row_order = np.array([sums[p] for p in sorted(sums)])
    val = X.val.cpu().numpy()
    assert np.array_equal(val, row_order)
    # scipy sums three or more duplicates of a pair in the order of its own (unstable) index sort: the last bit may differ
    assert np.all(np.abs(val - ref.data) <= 4 * np.finfo(np.float64).eps * np.abs(ref.data))
    rt = po.interaction_matrix(i, u, np.ones(len(u)), I, U)
    assert np.array_equal(X.t_ptr.cpu().numpy(), rt.indptr) and np.array_equal(X.t_col.cpu().numpy(), rt.indices)
    Xh = sp.csr_matrix((val, X.col.cpu().numpy(), X.row_ptr.cpu().numpy()), shape=(U, I)).T.tocsr()
    Xh.sort_indices()
    assert np.array_equal(X.t_val.cpu().numpy(), Xh.data)         # X^T holds X's values


# ------------------------------------------------------------------ SpMM
@pytest.mark.parametrize("U,I,l", [(900, 600, 22), (3000, 1200, 160), (400, 300, 300), (1000, 50, 37)])
def test_spmm_both_directions(U, I, l):
    from daisyrec_b200 import ops
    u, i, v = _coo(U, I, 25 * U, 2, real=True)
    i[:6000 if I > 100 else 0] = 7                               # a row of X^T longer than the warp path takes
    X = _X(u, i, v, U, I)
    ref = po.interaction_matrix(u, i, v, U, I)
    rng = np.random.default_rng(3)
    for transposed, (M, n) in ((False, (ref, I)), (True, (ref.T.tocsr(), U))):
        Zh = rng.standard_normal((n, l))
        Z = ops.puresvd_panel(n, l, 'cuda')
        Z[:n, :l] = _d(Zh, np.float64)
        Y = ops.puresvd_panel(M.shape[0], l, 'cuda')
        Y.fill_(7.0)
        ops.puresvd_spmm(X.operand(transposed), Z, l, Y)
        Yh = Y.cpu().numpy()
        want = M @ Zh
        bound = abs(M) @ np.abs(Zh)
        assert np.all(np.abs(Yh[:M.shape[0], :l] - want) <= 1e-13 * bound)
        assert np.all(Yh[:M.shape[0], l:] == 0)
        Y2 = torch.zeros_like(Y)
        ops.puresvd_spmm(X.operand(transposed), Z, l, Y2)
        assert torch.equal(Y2[:M.shape[0]], Y[:M.shape[0]])      # bitwise run to run


# ------------------------------------------------------------------ orth
def _orth(Yh, want_r=True):
    from daisyrec_b200 import ops
    m, l = Yh.shape
    Y = ops.puresvd_panel(m, l, 'cuda')
    Y[:m, :l] = _d(Yh, np.float64)
    R = ops.puresvd_orth(Y, m, l, want_r=want_r)
    return Y, R


def _check_orth(Yh, Y, R):
    m, l = Yh.shape
    Q = Y[:m, :l]
    Rl = R[:l, :l]
    eye = torch.eye(l, dtype=torch.float64, device='cuda')
    assert (Q.T @ Q - eye).abs().max().item() <= 1e-13
    Yd = _d(Yh, np.float64)
    assert torch.linalg.norm(Q @ Rl - Yd).item() <= 1e-13 * torch.linalg.norm(Yd).item()
    assert torch.all(torch.tril(Rl, -1) == 0)
    assert torch.all(Y[m:] == 0) and torch.all(Y[:, l:] == 0)


@pytest.mark.parametrize("m,l", [(500, 16), (5000, 160), (3000, 64), (1100, 1024)])
def test_orth_random(m, l):
    Yh = np.random.default_rng(m + l).standard_normal((m, l))
    Y, R = _orth(Yh)
    _check_orth(Yh, Y, R)


def test_orth_ill_conditioned_shift():
    rng = np.random.default_rng(3)
    m, l = 2000, 16
    A, _ = np.linalg.qr(rng.standard_normal((m, l)))
    B, _ = np.linalg.qr(rng.standard_normal((l, l)))
    Yh = A @ np.diag(np.logspace(0, -10, l)) @ B                 # kappa = 1e10
    Y, R = _orth(Yh)
    _check_orth(Yh, Y, R)


def test_orth_ml20m_tall_shape_reproducible():
    m, l = 138493, 160
    Yh = np.random.default_rng(0).standard_normal((m, l))
    Y, R = _orth(Yh)
    _check_orth(Yh, Y, R)
    Y2, R2 = _orth(Yh)
    assert torch.equal(Y, Y2) and torch.equal(R, R2)


def test_orth_rank_deficient_raises():
    rng = np.random.default_rng(4)
    Yh = rng.standard_normal((800, 30))
    Yh[:, 17] = Yh[:, 3] * 2.0 - Yh[:, 9]
    with pytest.raises(np.linalg.LinAlgError):
        _orth(Yh)
    Yh[:, 17] = 0.0
    with pytest.raises(np.linalg.LinAlgError):
        _orth(Yh)


# ------------------------------------------------------------------ small SVD
@pytest.mark.parametrize("l", [16, 160, 1024])
def test_small_svd(l):
    from daisyrec_b200 import ops
    rng = np.random.default_rng(l)
    Rh = np.linalg.qr(rng.standard_normal((2 * l, l)))[1]         # the R of a Gaussian panel, as the fit's last orth gives
    ld = (l + 63) // 64 * 64
    R = torch.zeros((ld, ld), dtype=torch.float64, device='cuda')
    R[:l, :l] = _d(Rh, np.float64)
    s, UT, VT = ops.puresvd_small_svd(R, l)
    s, UT, VT = s.cpu().numpy(), UT.cpu().numpy()[:l, :l], VT.cpu().numpy()[:l, :l]
    want = np.linalg.svd(Rh.T, compute_uv=False)
    # each column takes about l rotations per sweep, and their rounding adds up: 1.5e-13 sigma_1 was measured at l = 1024
    bar = 1e-13 if l <= 160 else 4e-13
    assert np.all(np.abs(np.sort(s)[::-1] - want) <= bar * want[0])
    assert np.abs(UT @ UT.T - np.eye(l)).max() <= bar
    assert np.abs(VT @ VT.T - np.eye(l)).max() <= bar
    assert np.abs((UT.T * s) @ VT - Rh.T).max() <= bar * want[0]


# ------------------------------------------------------------------ the class against the reference's runs
def _fit(U, I, f, u, i, v, topk=10):
    from daisyrec_b200.model import PureSVD
    m = PureSVD(_config(user_num=U, item_num=I, factors=f, topk=topk))
    m.fit(pd.DataFrame({'user': u.astype(np.int64), 'item': i.astype(np.int64), 'rating': v.astype(np.float64)}))
    return m


def test_synthetic_cases_vs_reference():
    g = golden("puresvd")
    for k in range(int(g["n_synthetic"])):
        U, I, f, topk, deficient = (int(x) for x in g[f"s{k}_meta"])
        u, i, v = g[f"s{k}_u"], g[f"s{k}_i"], g[f"s{k}_v"]
        if deficient:
            with pytest.raises(np.linalg.LinAlgError):
                _fit(U, I, f, u, i, v, topk)
            continue
        m = _fit(U, I, f, u, i, v, topk)
        P, Qv, s = m.user_vec.cpu().numpy(), m.item_vec.cpu().numpy(), m.sigma.cpu().numpy()
        assert P.shape == (U, f) and Qv.shape == (I, f)
        check_factors(P, Qv, s, g[f"s{k}_user_vec"], g[f"s{k}_item_vec"], g[f"s{k}_sigma"])
        X = po.interaction_matrix(u.astype(np.int64), i.astype(np.int64), v.astype(np.float64), U, I)
        warm = np.diff(X.indptr) > 0
        assert np.all(P[~warm] == 0) and np.all(Qv[np.bincount(X.indices, minlength=I) == 0] == 0)
        users = np.arange(U)
        cands = g[f"s{k}_cands"].astype(np.int64)
        got = m.rank(_Loader(users, cands, bs=16))
        assert got.dtype == np.int64 and got.shape == (U, topk)
        assert np.array_equal(got[warm], g[f"s{k}_rank"][warm]), k
        assert np.array_equal(got[~warm], cands[~warm, :topk]), k
        for a, want in zip(g[f"s{k}_full_u"], g[f"s{k}_full"]):
            fr = m.full_rank(int(a))
            assert fr.dtype == np.int64 and fr.shape == (topk,) and np.array_equal(fr, want), k
        pred = np.array([m.predict(int(a), int(b)) for a, b in zip(users, cands[:, 0])])
        assert np.abs(pred - g[f"s{k}_predict"]).max() <= 1e-10, k


def test_fit_bitwise_reproducible_and_oracle():
    U, I = 3000, 1300
    u, i, v = _coo(U, I, 40000, 9, dups=500)
    m1, m2 = _fit(U, I, 40, u, i, v), _fit(U, I, 40, u, i, v)
    assert torch.equal(m1.user_vec, m2.user_vec) and torch.equal(m1.item_vec, m2.item_vec)
    assert torch.equal(m1.sigma, m2.sigma)
    X = po.interaction_matrix(u, i, v, U, I)
    P, Qv, s = po.fit(X, 40)
    check_factors(m1.user_vec.cpu().numpy(), m1.item_vec.cpu().numpy(), m1.sigma.cpu().numpy(), P, Qv, s[:40])


def test_refusals():
    from daisyrec_b200.model import PureSVD
    U, I = 100, 80
    u, i, v = _coo(U, I, 2000, 1)
    df = pd.DataFrame({'user': u, 'item': i, 'rating': v})
    with pytest.raises(NotImplementedError, match='min'):
        PureSVD(_config(factors=71)).fit(df)
    with pytest.raises(NotImplementedError, match='1024'):
        PureSVD(_config(user_num=3000, item_num=2000, factors=1015)).fit(df)
    m = PureSVD(_config())
    with pytest.raises(RuntimeError):
        m.predict(0, 0)
    with pytest.raises(RuntimeError):
        m.full_rank(0)
    m.fit(df)
    with pytest.raises(IndexError):
        m.predict(U, 0)
    with pytest.raises(IndexError):
        m.predict(0, I)
    with pytest.raises(IndexError):
        m.full_rank(-1)
    cands = np.tile(np.arange(20), (4, 1))
    cands[1, 3] = I
    with pytest.raises(IndexError):
        m.rank(_Loader(np.arange(4), cands))
    bad = df.copy()
    bad.loc[0, 'item'] = I
    with pytest.raises(ValueError):
        PureSVD(_config()).fit(bad)


def test_ml100k_driver_sequence():
    """test.py's puresvd branch on config 1's ml-100k split through the drop-in class: PureSVD(config).fit(train_set) ->
    build_candidates_set -> rank -> calc_ranking_results, and full_rank / predict, against the reference's run."""
    from daisyrec_b200.model.PureSVDRecommender import PureSVD
    from daisyrec_b200.utils.dataset import CandidatesDataset, get_dataloader
    from daisyrec_b200.utils.metrics import calc_ranking_results
    from daisyrec_b200.utils.utils import get_ur, build_candidates_set
    g, gs, gr = golden("puresvd"), golden("ml100k_sampler"), golden("ml100k_rank")
    U, I, topk, seed, stride, f = (int(x) for x in g["ml_meta"])
    train_set = pd.DataFrame({'user': gs["coo_u"].astype(np.int64), 'item': gs["coo_i"].astype(np.int64), 'rating': 1.0})
    off = np.concatenate([[0], np.cumsum(gr["gt_len"])])
    test_ur = {int(a): gr["gt_flat"][off[k]:off[k + 1]].tolist() for k, a in enumerate(gr["test_u"])}
    cfg = _config(user_num=U, item_num=I, topk=topk, factors=f, cand_num=1000, seed=seed)
    np.random.seed(seed); torch.manual_seed(seed)
    train_ur = get_ur(train_set)
    model = PureSVD(cfg)
    model.fit(train_set)
    X = po.interaction_matrix(gs["coo_u"], gs["coo_i"], np.ones(len(gs["coo_u"])), U, I)
    h = hashlib.sha256()
    for a in (X.indptr.astype(np.int64), X.indices.astype(np.int32), X.data.astype(np.float64)):
        h.update(np.ascontiguousarray(a).tobytes())
    assert h.digest() == g["ml_X_sha"].tobytes()
    P, Qv, s = model.user_vec.cpu().numpy(), model.item_vec.cpu().numpy(), model.sigma.cpu().numpy()
    assert np.all(np.abs(s[:f] - g["ml_sigma"]) <= 1e-12 * g["ml_sigma"])
    from test_puresvd_cpu import separated
    ok = separated(s, f)
    up, ip = np.concatenate([P[:2], P[::stride]]), np.concatenate([Qv[:2], Qv[::stride]])
    assert np.abs(up[:, ok] - g["ml_user_rows"][:, ok]).max() <= 1e-10
    assert np.abs(ip[:, ok] - g["ml_item_rows"][:, ok]).max() <= 1e-10 * g["ml_sigma"][0]
    test_u, test_ucands = build_candidates_set(test_ur, train_ur, cfg)
    cands = np.stack([np.asarray(c[1], np.int64) for c in test_ucands])
    assert hashlib.sha256(cands.tobytes()).digest() == g["ml_cands_sha"].tobytes()
    preds = model.rank(get_dataloader(CandidatesDataset(test_ucands), batch_size=128, shuffle=False, num_workers=0))
    warm = g["ml_warm"]
    assert preds.dtype == np.int64 and preds.shape == g["ml_rank"].shape
    assert np.array_equal(preds[warm], g["ml_rank"][warm])                    # all 110 warm test users
    assert np.array_equal(preds[~warm], cands[~warm, :topk])
    for u, want in zip(g["ml_full_u"], g["ml_full"]):
        fr = model.full_rank(int(u))
        assert fr.dtype == np.int64 and fr.shape == (topk,) and np.array_equal(fr, want)
    for (u, i), want in zip(g["ml_predict_pairs"], g["ml_predict"]):
        p = model.predict(int(u), int(i))
        assert isinstance(p, np.float64) and abs(p - want) <= 1e-10
    kcfg = dict(logger=logging.getLogger('t'), res_path=tempfile.mkdtemp() + '/', metrics=["recall", "mrr", "ndcg", "hit", "precision"],
                item_num=I, topk=topk)
    res = calc_ranking_results(test_ur, preds, test_u, kcfg)
    assert [int(c) for c in res.columns[1:]] == g["ml_kpi_ks"].tolist()
    np.testing.assert_allclose(res.values[:, 1:].astype(np.float64), g["ml_kpi_sub"], rtol=1e-12, atol=1e-12)
