"""The numpy restatement of UserKNNCF (oracle/userknn_oracle.py) against tests/golden/userknn.npz, the reference's own runs
(oracle/gen_userknn.py): w_sparse [U, U] for every similarity, normalize and shrink on three data sets, pred_mat entries
(summed over reverse neighbours), rank, full_rank, predict, and ml-100k on config 1's split."""
import numpy as np
import pytest

from conftest import golden
from oracle import knn_oracle as ko
from oracle import userknn_oracle as uo
from test_itemknn_cpu import CENTRED, EXACT_DATA, N_CFG, _cfg, _data, _gold_w, compare_columns


@pytest.mark.parametrize("d", [0, 1, 2])
def test_w_sparse_every_configuration(d):
    g = golden("userknn")
    U, I, topk, u, i, v = _data(g, d)
    for k in range(N_CFG):
        sim, nrm, sh, maxk = _cfg(g, k)
        _, W = uo.fit(u, i, v, U, I, sim, nrm, sh, maxk)
        ref = _gold_w(g, f"d{d}_c{k}", U)
        compare_columns(W, ref, d in EXACT_DATA and sim not in CENTRED, f"d{d} {sim} {nrm} {sh} {maxk}")


def as_neighbours(W, maxk):
    """The reference's csc w_sparse as knn_oracle.Neighbours (ids ascending per column)."""
    n = W.shape[1]
    idx, val = np.full((n, maxk), -1, np.int32), np.zeros((n, maxk), np.float32)
    cnt = np.diff(W.indptr).astype(np.int32)
    for c in range(n):
        s = slice(W.indptr[c], W.indptr[c + 1])
        idx[c, :cnt[c]], val[c, :cnt[c]] = W.indices[s], W.data[s]
    return ko.Neighbours(idx, val, cnt, np.full(n, np.nan, np.float32))


@pytest.mark.parametrize("d", [0, 1, 2])
def test_scores_rank_full_rank_predict(d):
    g = golden("userknn")
    U, I, topk, u, i, v = _data(g, d)
    cands = g[f"d{d}_cands"].astype(np.int64)
    users = np.arange(U)
    seen = 0
    for k in range(N_CFG):
        p = f"d{d}_c{k}"
        if p + "_rank" not in g.files:
            continue
        seen += 1
        sim, nrm, sh, maxk = _cfg(g, k)
        X, W = uo.fit(u, i, v, U, I, sim, nrm, sh, maxk)
        ref = g[p + "_scores"]
        # the summation order, on the reference's own W (its choice among equal weights at the cut is its own)
        s = uo.scores(X, as_neighbours(_gold_w(g, p, U), maxk), users[:24], cands[:24])
        if d in EXACT_DATA and sim not in CENTRED:
            assert np.array_equal(s, ref), p                     # integer data: every pred_mat entry bitwise
        else:
            assert np.allclose(s, ref, rtol=1e-5, atol=1e-6 * np.abs(ref).max()), p
        Wr = as_neighbours(_gold_w(g, p, U), maxk)
        ids, sc = uo.rank(X, Wr, users, cands, topk)
        sc_all = uo.scores(X, Wr, users, cands)
        pos = lambda r: np.argmax(cands[:, :, None] == r[:, None, :], axis=1)
        got = np.take_along_axis(sc_all, pos(g[p + "_rank"].astype(np.int64)), 1)
        assert np.array_equal(got, -np.sort(-sc_all, axis=1)[:, :topk]), p      # the same score sequence; ties its own way
        full, fs = uo.full_rank(X, Wr, users[:6], topk)
        ref_full = g[p + "_full"].astype(np.int64)
        assert np.array_equal(np.take_along_axis(fs, full, 1), np.take_along_axis(fs, ref_full, 1)), p
        pr = uo.scores(X, Wr, users, cands[:, :1]).ravel()
        assert np.array_equal(pr, g[p + "_predict"]) or not (d in EXACT_DATA and sim not in CENTRED), p
        assert np.allclose(pr, g[p + "_predict"], rtol=1e-5, atol=1e-9), p
    assert seen


def test_ml100k_w_sparse_columns_and_scores():
    g = golden("userknn")
    gs = golden("ml100k_sampler")
    U, I, topk, seed, stride, maxk, shrink = (int(x) for x in g["ml_meta"])
    X, W = uo.fit(gs["coo_u"], gs["coo_i"], np.ones(len(gs["coo_u"])), U, I, "cosine", True, shrink, maxk)
    assert np.array_equal(np.diff(g["ml_W_indptr"]), W.cnt)
    cols = np.arange(0, U, stride)
    import scipy.sparse as sp
    Wc = sp.csc_matrix((g["ml_Wc_data"], g["ml_Wc_indices"].astype(np.int32), g["ml_Wc_indptr"]), shape=(U, len(cols)))
    for c, col in enumerate(cols):
        s = slice(Wc.indptr[c], Wc.indptr[c + 1])
        assert np.array_equal(np.sort(W.val[col, :W.cnt[col]]), np.sort(Wc.data[s])), col
    test_u = g["ml_test_u"].astype(np.int64)
    pairs = g["ml_predict_pairs"]
    pr = np.array([uo.scores(X, W, [a], np.array([[b]]))[0, 0] for a, b in pairs])
    assert np.allclose(pr, g["ml_predict"], rtol=1e-6)
    rank = g["ml_rank"].astype(np.int64)
    s = np.concatenate([uo.scores(X, W, [a], rank[k:k + 1, :20]) for k, a in enumerate(test_u)])
    close = np.isclose(s, g["ml_rank_scores"], rtol=1e-6).all(1)
    assert close.mean() >= 0.95                                  # W's ties at the cut move the rest
