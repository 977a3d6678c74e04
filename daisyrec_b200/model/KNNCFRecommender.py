"""ItemKNN on the GPU path, with the reference's class name, config keys and methods (daisy/model/KNNCFRecommender.py:380-457).

fit(train_set) has no training loop: X from the DataFrame, the similarity's value transform, the Gram matrix of the
transformed values, and per item column the maxk largest similarity weights (csrc/itemknn.cu on csrc/ease.cu's CSR and Gram).

    fit        -> drb_csr_build + drb_skipgram_group + drb_ease_csr, drb_itemknn_transform + drb_ease_scale, drb_ease_gram,
                  drb_itemknn_neighbours
    rank / full_rank / predict -> drb_itemknn_scores (+ drb_itemknn_topk)

The reference materialises pred_mat = X W as a lil_matrix; here it is NOT materialised: the model keeps X and at most maxk
neighbours per item, and an entry pred_mat[u, c] = sum_{i in N(c)} x_ui W[i, c] is summed when it is asked for, in fp64 over
ascending i (the order scipy's csc product adds in).

Neighbour selection: per column the min(maxk, item_num) largest weights by (weight descending, item id ascending), then exact
zeros dropped.  The reference's argpartition leaves the choice among equal weights at the cut unspecified; the id order is this
implementation's rule.  Negative weights (pearson, adjusted) are kept when they reach the top maxk.
"""
import numpy as np
import scipy.sparse as sp
import torch

from .. import ops
from .AbstractRecommender import NeighbourScorer


class ItemKNNCF(NeighbourScorer):
    MULTI_GPU = '{} runs on a single GPU'

    def __init__(self, config):
        """Same keys as the reference (KNNCFRecommender.py:402-411): user_num, item_num, maxk, shrink, normalize, similarity,
        topk (+ gpu, logger).  The DataFrame columns are 'user', 'item', 'rating' as convert_df hard-codes them (:36-38)."""
        super().__init__(config)
        self.user_num = config['user_num']
        self.item_num = config['item_num']
        self.k = config['maxk']
        self.shrink = config['shrink']
        self.normalize = config['normalize']
        self.similarity = config['similarity']
        self.topk = config['topk']
        self._X = self._W = self._w_host = None

    # ------------------------------------------------------------------ fit
    def fit(self, train_set):
        """KNNCFRecommender.py:415-432 on the device.  MemoryError when the fp64 [I, I] Gram matrix and its workspace do not
        fit in the free device memory."""
        if self.similarity not in ops.KNN_SIMILARITY:
            raise ValueError(f"value for parameter 'similarity' not recognized. Allowed values are: 'cosine', 'pearson', "
                             f"'adjusted', 'asymmetric', 'jaccard', 'tanimoto', 'dice', 'tversky'. Passed value was "
                             f"'{self.similarity}'")
        maxk = int(self.k)
        if not 1 <= maxk <= 1024:
            raise NotImplementedError(f'ItemKNNCF keeps 1 to 1024 neighbours per item on the GPU path; got maxk = {self.k}')
        u = np.asarray(train_set['user'].values)
        i = np.asarray(train_set['item'].values)
        v = np.array(train_set['rating'].values, dtype=np.float64)
        # scipy's coo checks (csc_matrix((ratings, (rows, cols)), shape)), before anything reaches the device
        for ids, hi, what in ((u, self.user_num, 'row'), (i, self.item_num, 'column')):
            if len(ids) and ids.max() >= hi:
                raise ValueError(f'{what} index exceeds matrix dimensions')
            if len(ids) and ids.min() < 0:
                raise ValueError(f'negative {what} index found')
        n = self.item_num
        self._X = self._W = self._w_host = None            # free the previous fit before the n x n allocation
        torch.cuda.empty_cache()
        free = torch.cuda.mem_get_info(self.device)[0]
        # the Gram matrix, the larger (fp64) of the two workspaces, X and its transformed copy, the neighbour arrays
        need = (8 * n * n + ops.L.lib().drb_ease_workspace_bytes(self.user_num, n, -1) + 40 * len(u) + 8 * self.user_num
                + (8 * maxk + 64) * n)
        if need > free:
            raise MemoryError(f'ItemKNNCF.fit needs {need} bytes of device memory for {n} items (the dense fp64 Gram matrix '
                              f'alone is {8 * n * n}); {free} bytes are free')
        d_u = torch.from_numpy(u.astype(np.int32)).to(self.device)
        d_i = torch.from_numpy(i.astype(np.int32)).to(self.device)
        d_v = torch.from_numpy(np.ascontiguousarray(v)).to(self.device)
        X = ops.ease_csr(d_u, d_i, d_v, self.user_num, n)
        del d_u, d_i, d_v
        Xt, ss, item_ptr = ops.itemknn_transform(X, self.similarity)
        cold = int((item_ptr[1:] == item_ptr[:-1]).sum())
        if cold:
            self.logger.info(f"ItemKNNCFRecommender: Detected {cold} ({cold / n * 100:.2f} %) cold items.")
        ws = ops.ease_workspace(Xt)
        G = ops.ease_gram(Xt, 0.0, ws)
        del ws, Xt
        self._W = ops.itemknn_neighbours(G, ss, self.similarity, self.normalize, self.shrink, maxk)
        del G
        self._X = X

    @property
    def w_sparse(self):
        """W as the reference builds it: scipy csc_matrix float32 [I, I], column c holding the neighbours of item c (built on
        first use)."""
        if self._w_host is None:
            self._w_host = self._neighbour_csc()
        return self._w_host

    # ------------------------------------------------------------------ scoring
    def predict(self, u, i):
        """-> numpy.float64: pred_mat[u, i] (KNNCFRecommender.py:434-438)."""
        if u >= self.user_num or i >= self.item_num:
            raise ValueError('User and/or item is unkown.')
        return self._predict_score(u, i)

    def rank(self, test_loader):
        """-> int64 ndarray [n_test_users, topk] of candidate ids by pred_mat[u, c], ties by candidate position
        (KNNCFRecommender.py:440-452)."""
        return super().rank(test_loader)

    def full_rank(self, u):
        """-> int64 ndarray [topk] of the top items of user u; no masking of train items (KNNCFRecommender.py:454-457)."""
        return super().full_rank(u)


class UserKNNCF(NeighbourScorer):
    """UserKNN on the GPU path (KNNCFRecommender.py:459-536): ItemKNN's similarity on X^T [I, U], whose columns are users.

    fit        -> drb_csr_build (X and X^T) + drb_ease_csr, drb_userknn_transpose + drb_itemknn_transform + drb_ease_scale,
                  drb_gram_image, per panel of users drb_gram_panel + drb_knn_neighbours_panel, drb_userknn_pairs +
                  drb_csr_build + drb_userknn_place (the reverse lists)
    rank / predict -> drb_userknn_scores (+ drb_itemknn_topk);  full_rank -> drb_userknn_full_scores + drb_itemknn_topk

    W is [U, U] with column j holding the neighbours of user j, and the reference's pred_mat = W X multiplies from the left:
    pred_mat[u, c] = sum_v W[u, v] x_vc, where W[u, v] != 0 exactly when u is one of v's neighbours.  So a user's scores sum
    over its reverse neighbours R(u) = {v : u in N(v)}, which fit keeps as a CSR over u; there is no bound on |R(u)|.  As in
    ItemKNNCF, pred_mat is not materialised: an entry is summed when asked for, in fp64 over ascending v (the order scipy's csc
    product adds in), from X in fp32 (the values convert_df's matrix holds, rounded once).

    The [U, U] Gram matrix is never held whole: one dense image of X (users x items; s8 when the exact-Gram rule holds per
    user, else fp64) stays resident, and the Gram is formed a panel of users at a time, each panel's rows selected before the
    next is formed.  The panel is the largest multiple of 128 users that fits in the free memory left after everything else,
    at most ops.USERKNN_PANEL_BYTES; ``_panel`` overrides it.

    The "cold users" line of fit is the reference's: its count comes from train.tocsc(), so it counts the items without rows.
    Neighbour selection and its tie rule are ItemKNNCF's (weight descending, user id ascending at the cut).
    """
    MULTI_GPU = '{} runs on a single GPU'

    def __init__(self, config):
        """Same keys as the reference (KNNCFRecommender.py:460-488): user_num, item_num, maxk, shrink, normalize, similarity,
        topk (+ gpu, logger).  The DataFrame columns are 'user', 'item', 'rating' as convert_df hard-codes them."""
        super().__init__(config)
        self.user_num = config['user_num']
        self.item_num = config['item_num']
        self.k = config['maxk']
        self.shrink = config['shrink']
        self.normalize = config['normalize']
        self.similarity = config['similarity']
        self.topk = config['topk']
        self._X = self._W = self._R = self._w_host = None
        self._panel = None

    def _need_resident(self, nnz):
        """Device bytes of X and X^T with the transform's copies and workspaces (built first, before the image)."""
        U, I = self.user_num, self.item_num
        return 40 * nnz + ops.L.lib().drb_ease_csr_workspace_bytes(max(U, I), nnz) + 16 * (U + I)

    def _need_rest(self, maxk, image):
        """Device bytes allocated after X^T: the image, one Gram panel of 128 users, the forward lists, and the reverse
        lists' pairs and CSR build."""
        U = self.user_num
        return image + 8 * 128 * U + 24 * U * maxk + ops.L.lib().drb_csr_workspace_bytes(U + 1, U * maxk)

    def fit(self, train_set):
        """KNNCFRecommender.py:490-510 on the device.  MemoryError when the image of X, one panel of 128 users, X, X^T and the
        neighbour lists do not fit in the free device memory.  It is checked twice: before anything is allocated, for
        everything with the smaller (s8) image, and once X^T has chosen the path, for what is still to be allocated with that
        path's image against the memory then free."""
        if self.similarity not in ops.KNN_SIMILARITY:
            raise ValueError(f"value for parameter 'similarity' not recognized. Allowed values are: 'cosine', 'pearson', "
                             f"'adjusted', 'asymmetric', 'jaccard', 'tanimoto', 'dice', 'tversky'. Passed value was "
                             f"'{self.similarity}'")
        maxk = int(self.k)
        if not 1 <= maxk <= 1024:
            raise NotImplementedError(f'UserKNNCF keeps 1 to 1024 neighbours per user on the GPU path; got maxk = {self.k}')
        u = np.asarray(train_set['user'].values)
        i = np.asarray(train_set['item'].values)
        v = np.array(train_set['rating'].values, dtype=np.float64)
        for ids, hi, what in ((u, self.user_num, 'row'), (i, self.item_num, 'column')):
            if len(ids) and ids.max() >= hi:
                raise ValueError(f'{what} index exceeds matrix dimensions')
            if len(ids) and ids.min() < 0:
                raise ValueError(f'negative {what} index found')
        U, I = self.user_num, self.item_num
        self._X = self._W = self._R = self._w_host = None
        torch.cuda.empty_cache()
        lib = ops.L.lib()

        def check(need, scale):
            torch.cuda.empty_cache()       # blocks the caching allocator holds but does not use count as free
            free = torch.cuda.mem_get_info(self.device)[0]
            if need > free:
                raise MemoryError(f'UserKNNCF.fit needs {need} more bytes of device memory for {U} users x {I} items (the '
                                  f'dense image of X alone is {lib.drb_gram_image_bytes(I, U, scale)}); {free} bytes are free')

        check(self._need_resident(len(u)) + self._need_rest(maxk, lib.drb_gram_image_bytes(I, U, 0)), 0)
        d_u = torch.from_numpy(u.astype(np.int32)).to(self.device)
        d_i = torch.from_numpy(i.astype(np.int32)).to(self.device)
        d_v = torch.from_numpy(np.ascontiguousarray(v)).to(self.device)
        X = ops.ease_csr(d_u, d_i, d_v, U, I)
        del d_v
        Xt, ss = ops.userknn_transform(X, d_u, d_i, self.similarity)
        del d_u, d_i
        cold = int((Xt.row_ptr[1:] == Xt.row_ptr[:-1]).sum())
        if cold:
            self.logger.info(f"UserKNNCFRecommender: Detected {cold} ({cold / I * 100:.2f} %) cold users.")
        rest = self._need_rest(maxk, lib.drb_gram_image_bytes(I, U, Xt.scale))
        check(rest, Xt.scale)
        panel = self._panel
        if panel is None:
            free = torch.cuda.mem_get_info(self.device)[0]
            panel = max(128, ops.userknn_panel_rows(U, free - (rest - 8 * 128 * U)))
        self._W = ops.userknn_neighbours(Xt, ss, self.similarity, self.normalize, self.shrink, maxk, panel)
        del Xt, ss
        self._R = ops.userknn_reverse(self._W)
        self._X = X

    @property
    def w_sparse(self):
        """W as the reference builds it: scipy csc_matrix float32 [U, U], column j holding the neighbours of user j (built on
        first use)."""
        if self._w_host is None:
            self._w_host = self._neighbour_csc(self.user_num)
        return self._w_host

    # ------------------------------------------------------------------ scoring
    def _scoring(self):
        return self._R, ops.userknn_rank, ops.userknn_full_rank, ops.userknn_predict

    def predict(self, u, i):
        """-> numpy.float64: pred_mat[u, i] (KNNCFRecommender.py:512-516)."""
        if u >= self.user_num or i >= self.item_num:
            raise ValueError('User and/or item is unkown.')
        return self._predict_score(u, i)

    def rank(self, test_loader):
        """-> int64 ndarray [n_test_users, topk] of candidate ids by pred_mat[u, c], ties by candidate position
        (KNNCFRecommender.py:518-530); None for an empty loader."""
        return super().rank(test_loader)

    def full_rank(self, u):
        """-> int64 ndarray [topk] of the top items of user u by (score descending, id ascending); no masking of train items
        (KNNCFRecommender.py:532-536)."""
        return super().full_rank(u)
