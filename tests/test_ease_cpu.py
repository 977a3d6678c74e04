"""The numpy restatement of EASE (oracle/ease_oracle.py) against tests/golden/ease.npz, the reference's own runs
(oracle/gen_ease.py): B in full on the synthetic cases, the rank quirk and tie order, full_rank, predict, and ml-100k on config 1's
split (X, P's diagonal, rows of B, candidate sets, rank on every test user)."""
import hashlib

import numpy as np
import pytest

from conftest import golden
from oracle import ease_oracle as eo
from oracle import i2v_oracle as io


def _case(g, k):
    U, I, topk = (int(v) for v in g[f"s{k}_meta"])
    return U, I, topk, g[f"s{k}_u"], g[f"s{k}_i"], g[f"s{k}_v"], float(g[f"s{k}_reg"])


def _sha(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.digest()


@pytest.mark.parametrize("k,scale", [(0, 0), (1, 1), (2, -1), (3, 0)])
def test_synthetic_cases(k, scale):
    g = golden("ease")
    U, I, topk, u, i, v, reg = _case(g, k)
    X, G, P, B = eo.fit(u, i, v, U, I, reg)
    assert eo.exact_scale(X) == scale
    if scale >= 0:                                         # integer work: the Gram is exact, and so its integer image
        q = (X.astype(np.float64) * 2.0 ** scale).astype(np.int64)
        assert np.array_equal(G, (q.T @ q).toarray() * 2.0 ** (-2 * scale) + reg * np.eye(I))
    want_B = g[f"s{k}_B"]
    # real weights: the reference's Gram is an fp32 sparse product that rounds, the restatement's is exact
    assert np.abs(B - want_B).max() <= (1e-12 if scale >= 0 else 1e-6) * np.abs(want_B).max()
    users = np.arange(U)
    cands = g[f"s{k}_cands"].astype(np.int64)
    ids, s = eo.rank(X, want_B, users, cands, topk)
    assert np.array_equal(ids, g[f"s{k}_rank"])            # the quirk (rows of B) and the tie order, every row
    full, _ = eo.full_rank(X, want_B, users[:6], topk)
    assert np.array_equal(full, g[f"s{k}_full"])
    pred = np.array([eo.predict(X, want_B, int(a), int(b)) for a, b in zip(users, cands[:, 0])])
    assert np.allclose(pred, g[f"s{k}_predict"], rtol=1e-12, atol=1e-15)
    # the rank quirk is observable: scoring with B instead of B^T changes the lists
    alt = np.take_along_axis(cands, eo.topk_order(np.take_along_axis(eo.user_scores(X, want_B, users), cands, 1), topk), 1)
    assert not np.array_equal(alt, ids)


def test_case0_edges():
    g = golden("ease")
    U, I, topk, u, i, v, reg = _case(g, 0)
    assert len(np.unique(np.stack([u, i]), axis=1)[0]) < len(u)          # duplicate pairs with their own values
    assert I - 1 not in set(i.tolist()) and {0, 1}.isdisjoint(u.tolist())  # a cold item, users without rows
    B = g["s0_B"]
    assert np.all(B[I - 1] == 0) and np.all(B[:, I - 1] == 0)            # the cold item's row and column
    assert np.array_equal(g["s0_rank"][:2], g["s0_cands"][:2, :topk])    # all-zero rows: the first positions
    assert np.array_equal(g["s0_full"][:2], np.tile(np.arange(topk), (2, 1)))


def test_exact_scale_bounds():
    import scipy.sparse as sp
    X = sp.csr_matrix(np.array([[127.0, 0.25], [0.0, 1.0]], np.float32))
    assert eo.exact_scale(X) == -1                          # 127 * 2^2 > 127
    X = sp.csr_matrix(np.array([[31.0, 0.25], [0.0, 1.0]], np.float32))
    assert eo.exact_scale(X) == 2
    X = sp.csr_matrix(np.full((133200, 1), 127.0, np.float32))
    assert eo.exact_scale(X) == -1                          # column sum of squares reaches 2^31


def test_ml100k():
    g, gs, gr = golden("ease"), golden("ml100k_sampler"), golden("ml100k_rank")
    U, I, topk, seed, stride = (int(v) for v in g["ml_meta"])
    cu, ci = gs["coo_u"].astype(np.int64), gs["coo_i"].astype(np.int64)
    X, G, P, B = eo.fit(cu, ci, np.ones(len(cu)), U, I, float(g["ml_reg"]))
    X.sort_indices()
    assert _sha(X.indptr.astype(np.int64), X.indices.astype(np.int32), X.data.astype(np.float32)) == g["ml_X_sha"].tobytes()
    assert eo.exact_scale(X) == 0
    assert np.allclose(np.diag(P), g["ml_P_diag"], rtol=1e-12, atol=0)
    rows = np.concatenate([B[:2], B[::stride]])
    assert np.abs(rows - g["ml_B_rows"]).max() <= 1e-12 * np.abs(g["ml_B_rows"]).max()
    assert np.abs(B.sum(0) - g["ml_B_colsum"]).max() <= 1e-11 * np.abs(B).sum(0).max()
    # test.py:112 with the driver's seed, then rank on every test user (the lists are tie-free beyond the zero rows)
    ur = {}
    for a, b in zip(cu.tolist(), ci.tolist()):
        ur.setdefault(a, set()).add(b)
    off = np.concatenate([[0], np.cumsum(gr["gt_len"])])
    test_ur = {int(a): gr["gt_flat"][off[k]:off[k + 1]].tolist() for k, a in enumerate(gr["test_u"])}
    np.random.seed(seed)
    test_u, cands = io.build_candidates_set(test_ur, ur, I, 1000)
    assert _sha(cands) == g["ml_cands_sha"].tobytes()
    assert np.array_equal(test_u, g["ml_test_u"])
    ids, _ = eo.rank(X, B, np.array(test_u), cands, topk)
    assert np.array_equal(ids, g["ml_rank"])
    full, _ = eo.full_rank(X, B, g["ml_full_u"], topk)
    assert np.array_equal(full, g["ml_full"])
    pred = [eo.predict(X, B, int(a), int(b)) for a, b in g["ml_predict_pairs"]]
    assert np.allclose(pred, g["ml_predict"], rtol=1e-10, atol=1e-15)
