"""numpy / scipy restatement of SLiM (daisy/model/SLiMRecommender.py) in Gram form; no sklearn.

Item j's ElasticNet(alpha, l1_ratio=elastic, positive=True, fit_intercept=False) against y = X[:, j] with column j of X zeroed
minimises, times n_samples = U,

    f_j(w) = 1/2 w^T G w - q^T w + l1 sum(w) + 1/2 l2 |w|^2,  w >= 0, w_j = 0,
    G = X^T X, q = G[:, j], l1 = alpha elastic U, l2 = alpha (1 - elastic) U.

l2 > 0 makes f_j strongly convex (modulus l2), so |w - w*| <= sqrt(2 gap(w) / l2) for the duality gap below.
"""
import numpy as np
import scipy.sparse as sp


def penalties(alpha, elastic, U):
    return alpha * elastic * U, alpha * (1.0 - elastic) * U


def x_csc(U, I, u, i, v):
    """SLiMRecommender.py:148-157: float64 csc [U, I], duplicates summed."""
    return sp.csc_matrix((np.asarray(v, np.float64), (np.asarray(u), np.asarray(i))), shape=(U, I))


def gram(X):
    """G = X^T X as dense fp64 (exact on integer data below 2^53)."""
    return np.asarray((X.T @ X).toarray(), np.float64)


def gap(G, j, w, l1, l2):
    """Formulation-A duality gap of column j's fit at w (sklearn _cd_fast.pyx gap_enet_sparse, positive=True), unscaled (sklearn's
    dual_gap_ is this over U).  Feature j and empty features contribute X^T A = 0."""
    w = np.asarray(w, np.float64).copy()
    w[j] = 0.0
    q = G[:, j].copy()
    q[j] = 0.0
    yy = G[j, j]
    Gw = G @ w                     # w_j = 0: equal to G with row and column j zeroed, once entry j is zeroed
    Gw[j] = 0.0
    r2 = yy - 2.0 * (w @ q) + w @ Gw
    ry = yy - w @ q
    xta = q - Gw - l2 * w
    dmax = max(0.0, float(xta.max())) if len(xta) else 0.0
    quad = r2 + l2 * (w @ w)
    primal = 0.5 * quad + l1 * w.sum()
    scale = l1 / dmax if dmax > l1 else 1.0
    dual = -0.5 * scale * scale * quad + scale * ry
    return primal - dual


def solve(G, j, l1, l2, max_rounds=200):
    """The optimum of column j's fit by an active-set method: solve (G_SS + l2 I) w_S = q_S - l1 on the support guess S, drop
    non-positive coefficients, add coordinates whose gradient says they should enter; exact up to fp64 rounding."""
    n = G.shape[0]
    q = G[:, j].copy()
    q[j] = 0.0
    allowed = np.diag(G) > 0
    allowed[j] = False
    H = G.copy()
    H[j, :] = 0.0
    H[:, j] = 0.0
    S = allowed & (q > l1)
    w = np.zeros(n)
    scale = max(1.0, float(np.abs(q).max()) if n else 1.0)
    for _ in range(max_rounds):
        w = np.zeros(n)
        idx = np.flatnonzero(S)
        if len(idx):
            w[idx] = np.linalg.solve(H[np.ix_(idx, idx)] + l2 * np.eye(len(idx)), q[idx] - l1)
        neg = S & (w <= 0)
        if neg.any():
            # step back towards the last feasible point is not needed for a convex QP with few changes: drop the most negative
            k = idx[np.argmin(w[idx])]
            S[k] = False
            continue
        grad = q - H @ w - l2 * w - l1
        viol = allowed & ~S & (grad > 1e-13 * scale)
        if not viol.any():
            return w
        S[np.flatnonzero(viol)[np.argmax(grad[viol])]] = True
    raise RuntimeError(f'active set did not settle for column {j}')


def eps(gap_value, l2):
    """Certified distance to the optimum from a duality gap."""
    return np.sqrt(2.0 * max(float(gap_value), 0.0) / l2)


def select(w, topk):
    """SLiMRecommender.py:86-107 for one column's fp64 coefficients -> (ids ascending int32, values float32): the
    min(nnz - 1, topk) largest non-zero coefficients, ties at the cut by lower id (the reference's argpartition leaves it open)."""
    w = np.asarray(w, np.float64)
    nz = np.flatnonzero(w)
    keep = min(len(nz) - 1, topk)
    if keep <= 0:
        return np.zeros(0, np.int32), np.zeros(0, np.float32)
    order = np.lexsort((nz, -w[nz]))[:keep]
    ids = np.sort(nz[order])
    return ids.astype(np.int32), w[ids].astype(np.float32)


def w_sparse(Wcols, topk):
    """Wcols fp64 [I, I] with column j item j's coefficients -> the reference's float32 csr w_sparse."""
    I = Wcols.shape[1]
    rows, cols, vals = [], [], []
    for j in range(I):
        ids, v = select(Wcols[:, j], topk)
        rows.append(ids), cols.append(np.full(len(ids), j, np.int32)), vals.append(v)
    return sp.csr_matrix((np.concatenate(vals) if vals else np.zeros(0, np.float32),
                          (np.concatenate(rows) if rows else np.zeros(0, np.int32),
                           np.concatenate(cols) if cols else np.zeros(0, np.int32))), shape=(I, I), dtype=np.float32)


def a_tilde(X, W):
    """SLiMRecommender.py:123-124: train.tocsr().dot(w_sparse), float64, in scipy's summation order."""
    return X.tocsr().dot(W)


def rank(A, users, cands, topk):
    """Candidate ids by A_tilde descending, ties by candidate position (the reference's argsort is unstable)."""
    sc = np.asarray(A[np.asarray(users)[:, None], cands].toarray(), np.float64)
    o = np.argsort(-sc, axis=1, kind='stable')[:, :topk]
    return np.take_along_axis(cands, o, 1), sc


def full_rank(A, u, topk):
    sc = np.asarray(A[u, :].toarray(), np.float64).ravel()
    return np.argsort(-sc, kind='stable')[:topk]
