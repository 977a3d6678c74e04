"""The numpy restatement of the device's PureSVD (oracle/puresvd_oracle.py: CholeskyQR3 normalisers, the projected SVD through
B^T = Q_b R, the user-side sign rule) against tests/golden/puresvd.npz, the reference's own sklearn runs
(oracle/gen_puresvd.py): sigma, factors, scores, rank, full_rank and predict on the synthetic cases and ml-100k."""
import hashlib

import numpy as np
import pytest

from conftest import golden
from oracle import i2v_oracle as io
from oracle import puresvd_oracle as po


def _case(g, k):
    U, I, f, topk, deficient = (int(v) for v in g[f"s{k}_meta"])
    u, i, v = g[f"s{k}_u"].astype(np.int64), g[f"s{k}_i"].astype(np.int64), g[f"s{k}_v"].astype(np.float64)
    return U, I, f, topk, bool(deficient), po.interaction_matrix(u, i, v, U, I)


def separated(sigma, k, rel=1e-6):
    """columns c < k whose sigma is >= rel (relative) away from both neighbours in the full spectrum ``sigma``."""
    s = np.asarray(sigma)
    ok = np.ones(k, bool)
    for c in range(k):
        for d in (c - 1, c + 1):
            if 0 <= d < len(s) and abs(s[c] - s[d]) < rel * s[c]:
                ok[c] = False
    return ok


def check_factors(user_vec, item_vec, sigma_full, want_user, want_item, want_sigma):
    """The parity bars of the issue-level contract: sigma 1e-12 relative, scores 1e-11, separated columns 1e-10 (user) and
    1e-10 sigma_1 (item)."""
    k = want_user.shape[1]
    assert np.all(np.abs(sigma_full[:k] - want_sigma) <= 1e-12 * want_sigma)
    S, W = user_vec @ item_vec.T, want_user @ want_item.T
    assert np.abs(S - W).max() <= 1e-11 * max(1.0, np.abs(W).max())
    ok = separated(sigma_full, k)
    assert ok.sum() >= k // 2
    assert np.abs(user_vec[:, ok] - want_user[:, ok]).max() <= 1e-10
    assert np.abs(item_vec[:, ok] - want_item[:, ok]).max() <= 1e-10 * want_sigma[0]


def _synthetic(g):
    return [k for k in range(int(g["n_synthetic"])) if not int(g[f"s{k}_meta"][4])]


@pytest.mark.parametrize("k", range(5))
def test_synthetic_cases(k):
    g = golden("puresvd")
    assert k in _synthetic(g)
    U, I, f, topk, _, X = _case(g, k)
    P, Qv, s = po.fit(X, f)
    check_factors(P, Qv, s, g[f"s{k}_user_vec"], g[f"s{k}_item_vec"], g[f"s{k}_sigma"])
    users = np.arange(U)
    cands = g[f"s{k}_cands"].astype(np.int64)
    ids, _ = po.rank(P, Qv, users, cands, topk)
    warm = np.diff(X.indptr) > 0
    assert np.array_equal(ids[warm], g[f"s{k}_rank"][warm])
    assert np.array_equal(ids[~warm], cands[~warm, :topk])              # exact zero rows: the candidate order
    full, _ = po.full_rank(P, Qv, g[f"s{k}_full_u"], topk)
    assert np.array_equal(full, g[f"s{k}_full"])
    pred = np.einsum("nk,nk->n", P[users], Qv[cands[:, 0]])
    assert np.abs(pred - g[f"s{k}_predict"]).max() <= 1e-10


def test_case_shapes():
    """the cases cover both branches of sklearn's transpose and n_iter rules, the l == min(U, I) edge and cold rows."""
    g = golden("puresvd")
    plans = {}
    for k in range(int(g["n_synthetic"])):
        U, I, f, _, deficient, X = _case(g, k)
        plans[k] = po.plan(U, I, f)
        if not deficient:
            assert np.linalg.matrix_rank(X.toarray()) >= f + 10
    assert plans[0][1:] == (7, False) and plans[1][1:] == (4, True)
    U, I, f, _, _, X = _case(g, 4)
    assert f + 10 == min(U, I) and np.all(np.diff(X.indptr) > 0) and np.all(np.bincount(X.indices, minlength=I) > 0)
    U, I, f, _, _, X = _case(g, 2)
    assert np.any(np.diff(X.indptr) == 0) and np.any(np.bincount(X.indices, minlength=I) == 0)
    assert X.nnz < len(g["s2_u"])                                       # duplicate pairs summed
    P, Qv, _ = po.fit(X, f)
    assert np.all(P[np.diff(X.indptr) == 0] == 0) and np.all(Qv[np.bincount(X.indices, minlength=I) == 0] == 0)


def test_rank_deficient_refused():
    g = golden("puresvd")
    k = [k for k in range(int(g["n_synthetic"])) if int(g[f"s{k}_meta"][4])][0]
    U, I, f, _, _, X = _case(g, k)
    with pytest.raises(np.linalg.LinAlgError):
        po.fit(X, f)


def test_cholqr3_shifted_ill_conditioned():
    rng = np.random.default_rng(3)
    m, l = 2000, 16
    A, _ = np.linalg.qr(rng.standard_normal((m, l)))
    B, _ = np.linalg.qr(rng.standard_normal((l, l)))
    Y = A @ np.diag(np.logspace(0, -10, l)) @ B                        # kappa = 1e10
    Q, R = po.cholqr3(Y)
    assert np.abs(Q.T @ Q - np.eye(l)).max() <= 1e-13
    assert np.linalg.norm(Q @ R - Y) <= 1e-13 * np.linalg.norm(Y)


def test_ml100k():
    g, gs, gr = golden("puresvd"), golden("ml100k_sampler"), golden("ml100k_rank")
    U, I, topk, seed, stride, f = (int(v) for v in g["ml_meta"])
    cu, ci = gs["coo_u"].astype(np.int64), gs["coo_i"].astype(np.int64)
    X = po.interaction_matrix(cu, ci, np.ones(len(cu)), U, I)
    h = hashlib.sha256()
    for a in (X.indptr.astype(np.int64), X.indices.astype(np.int32), X.data.astype(np.float64)):
        h.update(np.ascontiguousarray(a).tobytes())
    assert h.digest() == g["ml_X_sha"].tobytes()
    assert po.plan(U, I, f) == (160, 4, True)
    P, Qv, s = po.fit(X, f)
    assert np.all(np.abs(s[:f] - g["ml_sigma"]) <= 1e-12 * g["ml_sigma"])
    ok = separated(s, f)
    up, ip = np.concatenate([P[:2], P[::stride]]), np.concatenate([Qv[:2], Qv[::stride]])
    assert np.abs(up[:, ok] - g["ml_user_rows"][:, ok]).max() <= 1e-10
    assert np.abs(ip[:, ok] - g["ml_item_rows"][:, ok]).max() <= 1e-10 * g["ml_sigma"][0]
    assert np.abs(P.sum(0)[ok] - g["ml_user_colsum"][ok]).max() <= 1e-10 * U
    assert np.abs(Qv.sum(0)[ok] - g["ml_item_colsum"][ok]).max() <= 1e-10 * I * g["ml_sigma"][0]
    ur = {}
    for a, b in zip(cu.tolist(), ci.tolist()):
        ur.setdefault(a, set()).add(b)
    off = np.concatenate([[0], np.cumsum(gr["gt_len"])])
    test_ur = {int(a): gr["gt_flat"][off[k]:off[k + 1]].tolist() for k, a in enumerate(gr["test_u"])}
    np.random.seed(seed)
    test_u, cands = io.build_candidates_set(test_ur, ur, I, 1000)
    assert hashlib.sha256(cands.tobytes()).digest() == g["ml_cands_sha"].tobytes()
    warm = g["ml_warm"]
    assert np.array_equal(warm, np.diff(X.indptr)[test_u] > 0) and warm.sum() == 110
    ids, _ = po.rank(P, Qv, np.array(test_u), cands, topk)
    assert np.array_equal(ids[warm], g["ml_rank"][warm])                # every warm test user
    assert np.array_equal(ids[~warm], cands[~warm, :topk])
    full, _ = po.full_rank(P, Qv, g["ml_full_u"], topk)
    assert np.array_equal(full, g["ml_full"])
    pred = [P[a] @ Qv[b] for a, b in g["ml_predict_pairs"]]
    assert np.abs(np.array(pred) - g["ml_predict"]).max() <= 1e-10
