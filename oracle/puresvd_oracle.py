"""numpy / scipy restatement of PureSVD as the device computes it (csrc/puresvd.cu); no sklearn, no reference import.

The reference (daisy/model/PureSVDRecommender.py) calls sklearn's randomized_svd(X, factors, random_state=2019): l = factors + 10
random directions, n_iter = 7 if factors < 0.1 min(U, I) else 4 power rounds normalised by LU, a final QR, the SVD of
B = Q^T A and svd_flip.  The device keeps the algorithm and changes the normaliser: every panel is orthonormalised by shifted
CholeskyQR3, which spans the same subspace as LU or QR.  The projected SVD is taken as B^T = A^T Q = Q_b R (CholeskyQR3 again)
and the SVD of R^T = Ur S Vr^T, so that U_A = Q Ur and V_A = Q_b Vr.

    A = X^T when U < I (sklearn's transpose rule), else X.  Omega = RandomState(2019).normal(size=(min(U, I), l)).
    signs: every column of the user-side factor has its largest-magnitude entry (first index on ties) positive.
    user_vec = user side [:, :k], item_vec = item side [:, :k] * sigma.
"""
import numpy as np
import scipy.linalg as sl
import scipy.sparse as sp

U_ROUND = 2.0 ** -53
SEED = 2019


def interaction_matrix(u, i, v, U, I):
    """csr_matrix((rating, (user, item)), (U, I)) in fp64: duplicates summed, indices sorted."""
    X = sp.csr_matrix((np.asarray(v, np.float64), (np.asarray(u), np.asarray(i))), shape=(U, I))
    X.sum_duplicates()
    X.sort_indices()
    return X


def plan(U, I, factors):
    """-> (l, n_iter, transposed) of sklearn's randomized_svd defaults."""
    n = min(U, I)
    return factors + 10, (7 if factors < 0.1 * n else 4), U < I


def omega(U, I, l):
    return np.random.RandomState(SEED).normal(size=(min(U, I), l))


def cholqr(Y, shift):
    """One CholeskyQR pass: W = Y^T Y (+ s I), R = chol(W) upper, Y R^-1.  LinAlgError on a pivot <= l u max diag(W)."""
    m, l = Y.shape
    W = Y.T @ Y
    d = np.diag(W).copy()
    tau = l * U_ROUND * d.max()
    if shift:
        W = W + 11.0 * (m * l + l * (l + 1)) * U_ROUND * d.sum() * np.eye(l)
    try:
        R = np.linalg.cholesky(W).T
    except np.linalg.LinAlgError:
        raise np.linalg.LinAlgError("CholeskyQR: the panel is rank deficient") from None
    if not np.all(np.diag(R) ** 2 > tau):
        raise np.linalg.LinAlgError("CholeskyQR: the panel is rank deficient")
    return Y @ sl.solve_triangular(R, np.eye(l)), R


def cholqr3(Y):
    """Shifted CholeskyQR3 -> (Q, R) with Y = Q R: a shifted pass, then two plain ones."""
    Q, R1 = cholqr(Y, True)
    Q, R2 = cholqr(Q, False)
    Q, R3 = cholqr(Q, False)
    return Q, R3 @ R2 @ R1


def sign_rule(user_side):
    """+1 / -1 per column: the sign of each column's largest-magnitude entry (first index on ties)."""
    idx = np.argmax(np.abs(user_side), axis=0)
    s = np.sign(user_side[idx, np.arange(user_side.shape[1])])
    return np.where(s < 0, -1.0, 1.0)


def fit(X, factors, Om=None):
    """-> (user_vec [U, k], item_vec [I, k], sigma [l]) as the device computes them."""
    U, I = X.shape
    l, n_iter, transposed = plan(U, I, factors)
    A = (X.T if transposed else X).tocsr()
    At = A.T.tocsr()
    Z = omega(U, I, l) if Om is None else Om
    for _ in range(n_iter):
        Y, _ = cholqr3(A @ Z)
        Z, _ = cholqr3(At @ Y)
    Q, _ = cholqr3(A @ Z)
    Qb, R = cholqr3(At @ Q)
    Ur, s, Vrt = np.linalg.svd(R.T)
    order = np.argsort(-s, kind="stable")
    s, Ur, Vr = s[order], Ur[:, order], Vrt.T[:, order]
    UA, VA = Q @ Ur, Qb @ Vr
    user, item = (VA, UA) if transposed else (UA, VA)
    sg = sign_rule(user)
    user, item = user * sg, item * sg
    return user[:, :factors], (item * s)[:, :factors], s


def topk_order(s, k):
    """positions of the top k by (score descending, position ascending)."""
    return np.argsort(-s, axis=1, kind="stable")[:, :k]


def scores(user_vec, item_vec, users, cands=None):
    P = user_vec[np.asarray(users)]
    if cands is None:
        return P @ item_vec.T
    return np.einsum("nk,nck->nc", P, item_vec[np.asarray(cands)])


def rank(user_vec, item_vec, users, cands, topk):
    s = scores(user_vec, item_vec, users, cands)
    return np.take_along_axis(np.asarray(cands), topk_order(s, topk), 1), s


def full_rank(user_vec, item_vec, users, topk):
    s = scores(user_vec, item_vec, users)
    return topk_order(s, topk), s
