"""The numpy restatement of ItemKNNCF (oracle/knn_oracle.py) against tests/golden/itemknn.npz, the reference's own runs
(oracle/gen_itemknn.py): w_sparse for every similarity, normalize and shrink on three data sets, pred_mat entries, rank, full_rank,
predict, and ml-100k on config 1's split."""
import hashlib

import numpy as np
import pytest
import scipy.sparse as sp

from conftest import golden
from oracle import i2v_oracle as io
from oracle import knn_oracle as ko

N_CFG = 25
EXACT_DATA = (0, 1)                       # stars and binary: every formula but the mean-centred ones is bitwise
CENTRED = ('adjusted', 'pearson')


def _data(g, d):
    U, I, topk = (int(v) for v in g[f"d{d}_meta"])
    return U, I, topk, g[f"d{d}_u"].astype(np.int64), g[f"d{d}_i"].astype(np.int64), g[f"d{d}_v"]


def _cfg(g, k):
    return str(g["cfg_sim"][k]), bool(g["cfg_normalize"][k]), int(g["cfg_shrink"][k]), int(g["cfg_maxk"][k])


def _gold_w(g, p, n):
    return sp.csc_matrix((g[p + "_data"], g[p + "_indices"].astype(np.int32), g[p + "_indptr"]), shape=(n, n))


def compare_columns(W, ref, bitwise, where=""):
    """W (knn_oracle.Neighbours of every column) against the reference's csc ``ref``: per column the same number of
    neighbours and the same values in descending order; the same ids wherever the value differs from the first weight left
    out (the reference's argpartition decides ties at the cut its own way)."""
    for c in range(ref.shape[1]):
        s = slice(ref.indptr[c], ref.indptr[c + 1])
        rid, rv = ref.indices[s], ref.data[s]
        gid, gv = W.idx[c, :W.cnt[c]], W.val[c, :W.cnt[c]]
        assert len(gid) == len(rid), (where, c)
        if bitwise:
            assert np.array_equal(np.sort(gv), np.sort(rv)), (where, c)
            clear = lambda ids, v: set(ids[v != W.cut[c]].tolist())
            assert clear(gid, gv) == clear(rid, rv), (where, c)
        else:
            scale = np.abs(rv).max(initial=0)
            assert np.allclose(-np.sort(-gv), -np.sort(-rv), rtol=1e-6, atol=1e-6 * scale), (where, c)


@pytest.mark.parametrize("d", [0, 1, 2])
def test_w_sparse_every_configuration(d):
    g = golden("itemknn")
    U, I, topk, u, i, v = _data(g, d)
    assert len(g["cfg_sim"]) == N_CFG and set(g["cfg_sim"].tolist()) == set(ko.SIMILARITIES)
    X = ko.interaction_matrix(u, i, v, U, I)
    for k in range(N_CFG):
        sim, nrm, sh, maxk = _cfg(g, k)
        W = ko.neighbours(X, sim, nrm, sh, maxk)
        ref = _gold_w(g, f"d{d}_c{k}", I)
        assert ref.dtype == np.float32
        compare_columns(W, ref, d in EXACT_DATA and sim not in CENTRED, (d, sim, nrm, sh, maxk))


def test_asymmetric_is_cosine_and_jaccard_is_tanimoto():
    g = golden("itemknn")
    cfgs = [_cfg(g, k) for k in range(N_CFG)]
    for a, b in (("asymmetric", "cosine"), ("jaccard", "tanimoto")):
        for k, (sim, nrm, sh, maxk) in enumerate(cfgs):
            if sim == a:
                k2 = cfgs.index((b, nrm, sh, maxk))
                for d in range(3):
                    assert np.array_equal(g[f"d{d}_c{k}_data"], g[f"d{d}_c{k2}_data"])
                    assert np.array_equal(g[f"d{d}_c{k}_indices"], g[f"d{d}_c{k2}_indices"])


def test_data_set_edges():
    g = golden("itemknn")
    U, I, topk, u, i, v = _data(g, 0)
    assert len(np.unique(np.stack([u, i]), axis=1)[0]) < len(u)            # duplicate pairs
    assert I - 1 not in set(i.tolist()) and {0, 1}.isdisjoint(u.tolist())  # a cold item, users without rows
    W = _gold_w(g, "d0_c0", I)
    assert W[:, I - 1].nnz == 0 and W[I - 1].nnz == 0
    k600 = [k for k in range(N_CFG) if int(g["cfg_maxk"][k]) == 600][0]
    assert np.diff(g[f"d0_c{k600}_indptr"]).max() > 10                      # maxk >= I keeps every non-zero weight
    # negative weights survive when they reach the top maxk (pearson), zeros never do
    kp = [k for k in range(N_CFG) if _cfg(g, k) == ("pearson", True, 0, 10)][0]
    assert (g[f"d2_c{kp}_data"] != 0).all()


def same_ranking(ids, s, cands, want):
    """The reference ranks with an unstable argsort: its ids are ours on rows whose top k + 1 scores are distinct, and
    elsewhere the scores of its ids are the sorted top scores.  -> the number of rows compared by id."""
    k = want.shape[1]
    top = -np.sort(-s, axis=1)
    pos = np.stack([np.searchsorted(c, w, sorter=np.argsort(c)) for c, w in zip(cands, want)])
    pos = np.stack([np.argsort(c)[q] for c, q in zip(cands, pos)])
    assert np.array_equal(np.take_along_axis(cands, pos, 1), want)
    assert np.array_equal(np.take_along_axis(s, pos, 1), top[:, :k])
    clear = np.all(np.diff(top[:, :k + 1], axis=1) != 0, axis=1)
    assert np.array_equal(ids[clear], want[clear])
    return int(clear.sum())


@pytest.mark.parametrize("d", [0, 1, 2])
def test_scoring(d):
    g = golden("itemknn")
    U, I, topk, u, i, v = _data(g, d)
    X = ko.interaction_matrix(u, i, v, U, I)
    users = np.arange(U)
    cands = g[f"d{d}_cands"].astype(np.int64)
    seen = 0
    for k in range(N_CFG):
        p = f"d{d}_c{k}"
        if p + "_rank" not in g:
            continue
        seen += 1
        ref = _gold_w(g, p, I)                                # the reference's own W, so ties at the cut play no part
        cnt = np.diff(ref.indptr).astype(np.int32)
        idx = np.full((I, 10), -1, np.int32)
        val = np.zeros((I, 10), np.float32)
        for c in range(I):
            idx[c, :cnt[c]] = ref.indices[ref.indptr[c]:ref.indptr[c + 1]]
            val[c, :cnt[c]] = ref.data[ref.indptr[c]:ref.indptr[c + 1]]
        W = ko.Neighbours(idx, val, cnt, None)
        ids, s = ko.rank(X, W, users, cands, topk)
        want = g[p + "_scores"]
        assert want.dtype == np.float64
        if d in EXACT_DATA:                                   # x representable in fp32: the same sums in the same order
            assert np.array_equal(s[:24], want)
            same_ranking(ids, s, cands, g[p + "_rank"].astype(np.int64))
            fid, fs = ko.full_rank(X, W, users[:6], topk)
            same_ranking(fid, fs, np.tile(np.arange(I), (6, 1)), g[p + "_full"].astype(np.int64))
            assert np.array_equal(s[:, 0], g[p + "_predict"])
        else:                                                 # the reference multiplies the fp64 ratings, X is their fp32 rounding
            bound = ko.scores(X, W, users, cands, absolute=True)
            assert np.all(np.abs(s[:24] - want) <= 2e-7 * bound[:24])
            assert np.all(np.abs(s[:, 0] - g[p + "_predict"]) <= 2e-7 * bound[:, 0])
    assert seen == 4


def _sha(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.digest()


def ml100k_inputs():
    g, gs, gr = golden("itemknn"), golden("ml100k_sampler"), golden("ml100k_rank")
    cu, ci = gs["coo_u"].astype(np.int64), gs["coo_i"].astype(np.int64)
    off = np.concatenate([[0], np.cumsum(gr["gt_len"])])
    test_ur = {int(a): gr["gt_flat"][off[k]:off[k + 1]].tolist() for k, a in enumerate(gr["test_u"])}
    return g, cu, ci, test_ur


def sorted_columns(W):
    idx, val = W.indices.astype(np.int32).copy(), W.data.copy()
    for c in range(W.shape[1]):
        s = slice(W.indptr[c], W.indptr[c + 1])
        o = np.lexsort((idx[s], -val[s]))
        idx[s], val[s] = idx[s][o], val[s][o]
    return idx, val


def test_ml100k():
    g, cu, ci, test_ur = ml100k_inputs()
    U, I, topk, seed, stride, maxk, shrink = (int(v) for v in g["ml_meta"])
    X, W = ko.fit(cu, ci, np.ones(len(cu)), U, I, "cosine", True, shrink, maxk)
    Wc = W.csc(I)
    assert np.array_equal(Wc.indptr, g["ml_W_indptr"])
    idx, val = sorted_columns(Wc)
    assert _sha(Wc.indptr.astype(np.int64), val) == g["ml_W_val_sha"].tobytes()          # every weight, bitwise
    cols = np.arange(0, I, stride)
    ref = sp.csc_matrix((g["ml_Wc_data"], g["ml_Wc_indices"].astype(np.int32), g["ml_Wc_indptr"]), shape=(I, len(cols)))
    sub = ko.Neighbours(W.idx[cols], W.val[cols], W.cnt[cols], W.cut[cols])
    compare_columns(sub, ref, True, "ml-100k")
    ur = {}
    for a, b in zip(cu.tolist(), ci.tolist()):
        ur.setdefault(a, set()).add(b)
    np.random.seed(seed)
    test_u, cands = io.build_candidates_set(test_ur, ur, I, 1000)
    assert _sha(cands) == g["ml_cands_sha"].tobytes() and np.array_equal(test_u, g["ml_test_u"])
    ids, s = ko.rank(X, W, np.array(test_u), cands, topk)
    got = -np.sort(-s, axis=1)[:, :20]
    # 23 columns have equal weights at the cut and the reference's argpartition breaks those ties its own way, so the id digest
    # is not expected to match; what those columns and the unstable argsort of rank can reach is bounded instead
    assert np.array_equal(got, g["ml_rank_scores"])
    assert (ids == g["ml_rank"]).all(1).sum() >= 300
    assert np.array_equal(ko.full_rank(X, W, g["ml_full_u"], topk)[0], g["ml_full"])
    pred = ko.scores(X, W, g["ml_predict_pairs"][:, 0], g["ml_predict_pairs"][:, 1:2])[:, 0]
    assert np.array_equal(pred, g["ml_predict"])
