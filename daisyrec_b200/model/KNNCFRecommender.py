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
