"""numpy / scipy restatement of UserKNNCF (daisy/model/KNNCFRecommender.py:459-536) and MostPop (daisy/model/PopRecommender.py),
the references the GPU path is tested against.

UserKNN: knn_oracle's similarity on X^T [I, U] (its columns are users), so W is [U, U] with column v = N(v).  pred_mat = W X
(the reference multiplies from the left): pred[u, c] = sum_{v in R(u)} W[u, v] x_vc with R(u) = {v : u in N(v)}, summed in
fp64 over ascending v, the order of scipy's csc product (csr_matmat on the transposes).  Ties of a ranking by position.

MostPop: item_cnt = value_counts of the item column (every row), item_score = cnt / (1 + cnt) in fp64.
"""
import numpy as np

from oracle import knn_oracle as ko


def fit(u, i, v, user_num, item_num, similarity, normalize, shrink, maxk, cols=None):
    """-> (X csr float32 [U, I], Neighbours of the user columns ``cols`` (default: every user))."""
    X = ko.interaction_matrix(u, i, v, user_num, item_num)
    Xt = X.T.tocsr()
    Xt.sort_indices()
    return X, ko.neighbours(Xt, similarity, normalize, shrink, maxk, cols)


def scores(X, W, users, cands=None):
    """fp64 [n, C]: pred_mat[u, c] over ascending v; every item when cands is None."""
    U = X.shape[0]
    R = W.csc(U).tocsr()
    R.sort_indices()
    out = np.zeros((len(users), X.shape[1] if cands is None else cands.shape[1]), np.float64)
    for r, u in enumerate(users):
        vs, ws = R.indices[R.indptr[u]:R.indptr[u + 1]], R.data[R.indptr[u]:R.indptr[u + 1]].astype(np.float64)
        Xv = X[vs].toarray().astype(np.float64)
        if cands is not None:
            Xv = Xv[:, cands[r]]
        acc = np.zeros(out.shape[1], np.float64)
        for q in range(len(vs)):
            acc = acc + Xv[q] * ws[q]
        out[r] = acc
    return out


def rank(X, W, users, cands, k):
    s = scores(X, W, users, cands)
    return np.take_along_axis(cands, ko.topk_order(s, k), 1), s


def full_rank(X, W, users, k):
    s = scores(X, W, users)
    return ko.topk_order(s, k), s


def mostpop(items, item_num):
    """-> (item_cnt_ref fp64 [I], item_score fp64 [I])."""
    cnt = np.bincount(np.asarray(items, np.int64), minlength=item_num).astype(np.float64)
    return cnt, cnt / (1 + cnt)
