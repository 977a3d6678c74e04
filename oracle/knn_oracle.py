"""numpy / scipy restatement of ItemKNNCF (daisy/model/KNNCFRecommender.py:235-457), the reference the GPU path is tested
against.  Written from the formulas, in the reference's dtypes and evaluation order:

X     csr_matrix((ratings, (u, i))).astype(float32), duplicates summed in fp64 first.
X'    adjusted: minus the user's mean; pearson: minus the item's mean; jaccard / tanimoto / dice / tversky: every stored value 1.
      Means are fp32 sums in storage order (scipy's matvec) divided in fp64 and rounded to fp32.
ss    fp32 sum over each item of x'^2, in user order; its fp32 square root for cosine / asymmetric / adjusted / pearson.
g     X'^T X' computed exactly in fp64 and rounded to fp32 (what the reference's fp32 product gives on integer data).
w     fp32, left to right: normalised cosine family g * (1 / (ss_j ss_i + shrink + 1e-6)); tanimoto g * (1 / (ss_j + ss_i - g +
      shrink + 1e-6)); dice g * (1 / (ss_j + ss_i + shrink + 1e-6)); tversky (alpha = beta = 1) g * (1 / (g + (ss_j - g) +
      (ss_i - g) + shrink + 1e-6)); un-normalised cosine family g / shrink (g when shrink == 0).  w_jj = 0.  asymmetric with
      the class's alpha = 0.5 raises ss to the power 1.0: it is cosine.
N(j)  the min(maxk, I) largest w by (w descending, id ascending), exact zeros dropped, stored by ascending id.
score pred_mat[u, c] = sum_{i in N(c)} x_ui W[i, c] in fp64 over ascending i; ties of a ranking by position ascending.
"""
import numpy as np
import scipy.sparse as sp

BINARY = ('jaccard', 'tanimoto', 'dice', 'tversky')
SIMILARITIES = ('cosine', 'asymmetric', 'adjusted', 'pearson') + BINARY
F32 = np.float32


def interaction_matrix(u, i, v, user_num, item_num):
    X = sp.csr_matrix((np.asarray(v, np.float64), (u, i)), shape=(user_num, item_num)).astype(F32)
    X.sort_indices()
    return X


def _seq_sums(M):
    """fp32 row sums of a csr matrix in storage order."""
    return np.asarray(M @ np.ones(M.shape[1], F32), F32).ravel()


def _mean(sums, counts):
    m = np.zeros(len(sums), F32)
    nz = counts > 0
    m[nz] = (sums[nz].astype(np.float64) / counts[nz]).astype(F32)
    return m


def transform(X, similarity):
    """-> X' (csr float32, the structure of X)."""
    Xt = X.copy()
    counts = np.diff(X.indptr)
    if similarity == 'adjusted':
        Xt.data = Xt.data - np.repeat(_mean(_seq_sums(X), counts), counts)
    elif similarity == 'pearson':
        Xc = X.tocsc()
        Xc.sort_indices()
        n = np.diff(Xc.indptr)
        Xc.data = Xc.data - np.repeat(_mean(_seq_sums(sp.csr_matrix((Xc.data, Xc.indices, Xc.indptr), shape=X.shape[::-1])), n), n)
        Xt = Xc.tocsr()
        Xt.sort_indices()
    elif similarity in BINARY:
        Xt.data = np.ones_like(Xt.data)
    elif similarity not in SIMILARITIES:
        raise ValueError(similarity)
    return Xt


def sum_of_squared(Xt, similarity):
    Xc = Xt.tocsc()
    Xc.sort_indices()
    sq = sp.csr_matrix((Xc.data * Xc.data, Xc.indices, Xc.indptr), shape=Xt.shape[::-1])
    ss = _seq_sums(sq)
    return ss if similarity in BINARY else np.sqrt(ss)


def gram_columns(Xt, cols=None):
    """fp32 [I, len(cols)]: columns of X'^T X', each product and sum exact in fp64, rounded once."""
    Xd = Xt.astype(np.float64).tocsc()
    R = Xd if cols is None else Xd[:, cols]
    return np.asarray((Xd.T @ R).toarray(), np.float64).astype(F32)


def column_weights(g, ss, cols, similarity, normalize, shrink):
    """fp32 weights [I, len(cols)] of the columns ``cols`` from their Gram columns g (modified: w_jj = 0)."""
    cols = np.asarray(cols)
    g[cols, np.arange(len(cols))] = 0.0
    shrink, eps, one = F32(shrink), F32(1e-6), F32(1.0)
    ssi, ssj = ss[:, None], ss[cols][None, :]
    if similarity in ('tanimoto', 'jaccard'):
        d = ssj + ssi - g + shrink + eps
    elif similarity == 'dice':
        d = ssj + ssi + shrink + eps
    elif similarity == 'tversky':
        d = g + (ssj - g) + (ssi - g) + shrink + eps
    elif normalize:
        d = ssj * ssi + shrink + eps
    else:
        return g / shrink if shrink != 0 else g
    assert d.dtype == F32
    return g * (one / d)


class Neighbours:
    def __init__(self, idx, val, cnt, cut):
        self.idx, self.val, self.cnt, self.cut = idx, val, cnt, cut     # cut: the first weight left out (nan: none)

    def csc(self, n):
        keep = np.arange(self.idx.shape[1])[None, :] < self.cnt[:, None]
        return sp.csc_matrix((self.val[keep], self.idx[keep], np.concatenate([[0], np.cumsum(self.cnt)])), shape=(n, len(self.cnt)))


def select(w, maxk):
    """Top min(maxk, I) of each column of w by (w desc, id asc), zeros dropped, ids ascending -> Neighbours (padded arrays)."""
    n, m = w.shape
    keep = min(maxk, n)
    idx = np.full((m, maxk), -1, np.int32)
    val = np.zeros((m, maxk), F32)
    cnt = np.zeros(m, np.int32)
    cut = np.full(m, np.nan, F32)
    for c in range(m):
        col = w[:, c]
        order = np.argsort(-col, kind='stable')
        if keep < n:
            cut[c] = col[order[keep]]
        top = np.sort(order[:keep][col[order[:keep]] != 0])
        cnt[c] = len(top)
        idx[c, :len(top)] = top
        val[c, :len(top)] = col[top]
    return Neighbours(idx, val, cnt, cut)


def fit(u, i, v, user_num, item_num, similarity, normalize, shrink, maxk, cols=None):
    """-> (X, Neighbours of ``cols`` (default: every item))."""
    X = interaction_matrix(u, i, v, user_num, item_num)
    return X, neighbours(X, similarity, normalize, shrink, maxk, cols)


def neighbours(X, similarity, normalize, shrink, maxk, cols=None):
    Xt = transform(X, similarity)
    cols = np.arange(X.shape[1]) if cols is None else np.asarray(cols)
    w = column_weights(gram_columns(Xt, cols), sum_of_squared(Xt, similarity), cols, similarity, normalize, shrink)
    return select(w, maxk)


def scores(X, W, users, cands=None, absolute=False):
    """fp64 [n, C]: sum over q ascending of x[u, idx[c, q]] * val[c, q]; every item when cands is None.  ``absolute`` sums
    |x w| instead (the scale rounding errors are measured against)."""
    Xu = X[users].toarray().astype(np.float64)
    if cands is None:
        cands = np.tile(np.arange(X.shape[1]), (len(users), 1))
    val = W.val.astype(np.float64)
    acc = np.zeros(cands.shape, np.float64)
    for q in range(W.idx.shape[1]):
        iq = W.idx[cands, q]
        term = np.take_along_axis(Xu, np.maximum(iq, 0), 1) * np.where(iq >= 0, val[cands, q], 0.0)
        acc = acc + (np.abs(term) if absolute else term)
    return acc


def topk_order(s, k):
    return np.argsort(-s, axis=1, kind='stable')[:, :k]


def rank(X, W, users, cands, k):
    s = scores(X, W, users, cands)
    return np.take_along_axis(cands, topk_order(s, k), 1), s


def full_rank(X, W, users, k):
    s = scores(X, W, users)
    return topk_order(s, k), s
