"""The SLiM restatement in oracle/slim_oracle.py against the reference's own runs in tests/golden/slim.npz (oracle/gen_slim.py):
the Gram-form gap reproduces sklearn's dual_gap_, the reference's coefficients lie within their certified distance of the
oracle's optimum, the selection quirk reproduces w_sparse bit for bit, and A_tilde / rank / full_rank / predict follow."""
import hashlib

import numpy as np
import scipy.sparse as sp
from conftest import golden

from oracle import slim_oracle as so

INTEGER = (0, 1, 3)          # data sets with integer values: G and A_tilde exact


def _data(g, d):
    U, I = (int(v) for v in g[f"d{d}_meta"])
    return U, I, g[f"d{d}_u"].astype(np.int64), g[f"d{d}_i"].astype(np.int64), g[f"d{d}_v"]


def _sparse(g, p, I, cls=sp.csc_matrix, dtype=np.float64):
    return cls((g[p + "_data"].astype(dtype), g[p + "_indices"].astype(np.int32), g[p + "_indptr"]), shape=(I, I))


def _coef(g, p, I):
    return _sparse(g, p, I).toarray()


def _w(g, p, I):
    return _sparse(g, p + "_W", I, sp.csr_matrix, np.float32)


def cases():
    g = golden("slim")
    for d in range(int(g["n_data"])):
        for k, (alpha, elastic) in enumerate(g["configs"]):
            yield g, d, k, float(alpha), float(elastic)


def test_gap_matches_sklearn():
    for g, d, k, alpha, elastic in cases():
        U, I, u, i, v = _data(g, d)
        G = so.gram(so.x_csc(U, I, u, i, v))
        l1, l2 = so.penalties(alpha, elastic, U)
        for suffix in ("", "t"):
            W = _coef(g, f"d{d}_c{k}_coef{suffix}", I)
            ref = g[f"d{d}_c{k}_gap{suffix}"]
            for j in range(I):
                mine = so.gap(G, j, W[:, j], l1, l2) / U
                assert abs(mine - ref[j]) <= 1e-9 * abs(ref[j]) + 1e-13 * G[j, j] / U, (d, k, j, mine, ref[j])


def test_reference_within_certified_distance_of_optimum():
    for g, d, k, alpha, elastic in cases():
        U, I, u, i, v = _data(g, d)
        G = so.gram(so.x_csc(U, I, u, i, v))
        l1, l2 = so.penalties(alpha, elastic, U)
        for suffix in ("", "t"):
            W = _coef(g, f"d{d}_c{k}_coef{suffix}", I)
            gaps = g[f"d{d}_c{k}_gap{suffix}"] * U
            for j in range(I):
                w = so.solve(G, j, l1, l2)
                assert so.gap(G, j, w, l1, l2) <= 1e-10 * max(G[j, j], 1.0)
                dist = np.linalg.norm(W[:, j] - w)
                assert dist <= so.eps(gaps[j], l2) + 1e-7 * (1 + np.abs(w).max()), (d, k, j, suffix, dist)
                assert W[j, j] == 0 and np.all(W[:, j] >= 0)
    g = golden("slim")
    assert g["tight"][0] == 1e-10


def test_selection_reproduces_w_sparse():
    for g, d, k, alpha, elastic in cases():
        U, I, u, i, v = _data(g, d)
        W = _coef(g, f"d{d}_c{k}_coef", I)
        for t, topk in enumerate(g["topks"]):
            mine = so.w_sparse(W, int(topk))
            ref = _w(g, f"d{d}_c{k}_t{t}", I)
            assert mine.dtype == np.float32 and (mine != ref).nnz == 0, (d, k, t)
            # the quirk: a column with nnz <= topk keeps nnz - 1, one with nnz <= 1 nothing
            nnz = (W != 0).sum(0)
            kept = np.diff(ref.tocsc().indptr)
            assert np.array_equal(kept, np.clip(np.minimum(nnz - 1, int(topk)), 0, None))


def test_scores_rank_full_rank_predict():
    for g, d, k, alpha, elastic in cases():
        U, I, u, i, v = _data(g, d)
        X = so.x_csc(U, I, u, i, v)
        users = np.arange(U)
        cands = g[f"d{d}_cands"].astype(np.int64)
        for t, topk in enumerate(g["topks"]):
            p = f"d{d}_c{k}_t{t}"
            A = so.a_tilde(X, _w(g, p, I))
            if d in INTEGER:
                assert np.array_equal(A[:8].toarray(), g[p + "_A"])
            else:
                np.testing.assert_allclose(A[:8].toarray(), g[p + "_A"], rtol=1e-12, atol=1e-14)
            kk = min(int(topk), cands.shape[1])
            ids, sc = so.rank(A, users, cands, kk)
            ref = g[p + "_rank"].astype(np.int64)
            # ids are comparable where the top scores are tie-free; the scores of the returned ids always are
            top = -np.sort(-sc, axis=1)
            pos = [np.array([list(c).index(x) for x in r]) for c, r in zip(cands, ref)]
            ref_s = np.stack([s[q] for s, q in zip(sc, pos)])
            assert np.array_equal(ref_s, top[:, :kk])
            free = np.array([len(np.unique(row[:kk + 1])) == min(kk + 1, len(row)) for row in top])
            assert np.array_equal(ids[free], ref[free])
            for a in range(4):
                f = so.full_rank(A, a, int(topk))
                sa = np.asarray(A[a].toarray()).ravel()
                assert np.array_equal(np.sort(sa[f]), np.sort(sa[g[p + "_full"][a].astype(np.int64)]))
            pred = np.array([A[a, b] for a, b in zip(users[:8], cands[:8, 0])])
            assert np.array_equal(pred, g[p + "_predict"]) if d in INTEGER else np.allclose(pred, g[p + "_predict"], 1e-12, 1e-14)


def test_numpy_state_after_fit():
    g = golden("slim")
    for d in range(int(g["n_data"])):
        U, I, *_ = _data(g, d)
        np.random.seed(int(g["seed"]))
        np.random.randint(0, 2147483647, size=I)
        st = np.random.get_state()
        h = hashlib.sha256(np.asarray(st[1], np.uint32).tobytes() + np.array([st[2], st[3]], np.int64).tobytes()).digest()
        assert h == g[f"d{d}_c0_t0_rng"].tobytes()
