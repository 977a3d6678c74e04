"""numpy fp64 restatement of EASE (daisy/model/EASERecommender.py:30-74), the reference the GPU path is tested against.

fit: X = csr_matrix((values, (u, i))).astype(float32); G = X^T X + reg I in fp64 (exact for the s8-representable data the
reference's fp32 product also gets exactly); P = inv(G); B = -P / diag(P) with a zero diagonal.
rank scores candidates with ROWS of B (s_c = sum_i x_ui B[c, i]); full_rank and predict use x_u B.  Ties: score
descending, then candidate position (rank) or item id (full_rank) ascending.
"""
import numpy as np
import scipy.sparse as sp


def interaction_matrix(u, i, v, user_num, item_num):
    return sp.csr_matrix((np.asarray(v, np.float64), (u, i)), shape=(user_num, item_num)).astype(np.float32)


def gram(X, reg):
    Xd = X.astype(np.float64)
    return (Xd.T @ Xd).toarray() + reg * np.eye(X.shape[1])


def weights(P):
    B = -P / np.diag(P)
    np.fill_diagonal(B, 0.)
    return B


def fit(u, i, v, user_num, item_num, reg):
    """-> (X, G, P, B)"""
    X = interaction_matrix(u, i, v, user_num, item_num)
    G = gram(X, reg)
    P = np.linalg.inv(G)
    return X, G, P, weights(P)


def topk_order(scores, k):
    """Stable top-k of each row: score descending, then position ascending."""
    return np.argsort(-scores, axis=1, kind='stable')[:, :k]


def rank_scores(X, B, users, cands):
    Xu = X[users].toarray().astype(np.float64)                    # [n, I]
    return np.einsum('ni,nci->nc', Xu, B[cands])                  # rows of B


def rank(X, B, users, cands, k):
    s = rank_scores(X, B, users, cands)
    return np.take_along_axis(cands, topk_order(s, k), 1), s


def user_scores(X, B, users):
    return X[users].toarray().astype(np.float64) @ B


def full_rank(X, B, users, k):
    s = user_scores(X, B, users)
    return topk_order(s, k), s


def predict(X, B, u, i):
    return float((X[u].toarray().astype(np.float64) @ B[:, i]).item())


def exact_scale(X):
    """Smallest s in [0, 7] with every x 2^s an integer in [-127, 127] and max_i sum_u (x 2^s)^2 < 2^31, else -1."""
    x = X.data.astype(np.float64)
    for s in range(8):
        q = x * 2.0 ** s
        if np.all(q == np.round(q)):
            colsq = np.bincount(X.indices, weights=q * q, minlength=X.shape[1]) if len(q) else np.zeros(1)
            if np.abs(q).max(initial=0) <= 127 and colsq.max(initial=0) < 2.0 ** 31:
                return s
            return -1
    return -1
