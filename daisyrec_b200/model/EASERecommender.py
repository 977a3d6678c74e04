"""EASE on the GPU path, with the reference's class name, config keys and methods (daisy/model/EASERecommender.py:16-74).

fit(train_set) has no training loop: X from the DataFrame, G = X^T X + reg I, P = G^-1, B = -P / diag(P) with a zero
diagonal, all on the device in fp64 (csrc/ease.cu).  ``item_similarity`` is the device fp64 [I, I] tensor B.

    fit        -> drb_csr_build + drb_skipgram_group + drb_ease_csr, drb_ease_gram, drb_ease_inverse, drb_ease_weights
    rank       -> drb_ease_rank: s_c = sum_i x_ui B[c, i] -- the reference gathers ROWS of B for the candidates
                  (EASERecommender.py:62), i.e. it scores with B^T; kept as the reference computes it
    full_rank  -> drb_ease_full_rank: x_u B        predict -> drb_ease_predict: x_u . B[:, i]
"""
import numpy as np
import scipy.sparse as sp
import torch

from .. import ops
from .AbstractRecommender import DeviceRecommender


class EASE(DeviceRecommender):
    MULTI_GPU = '{} runs on a single GPU'

    def __init__(self, config):
        """Same keys as the reference (EASERecommender.py:17-28): reg, topk, user_num, item_num, UID_NAME, IID_NAME,
        INTER_NAME (+ gpu, logger)."""
        super().__init__(config)
        self.inter_name = config['INTER_NAME']
        self.iid_name = config['IID_NAME']
        self.uid_name = config['UID_NAME']
        self.user_num = config['user_num']
        self.item_num = config['item_num']
        self.reg_weight = config['reg']
        self.topk = config['topk']
        self.item_similarity = None
        self._X = None
        self._csr_host = None

    # ------------------------------------------------------------------ fit
    def fit(self, train_set):
        """EASERecommender.py:30-47 on the device.  numpy.linalg.LinAlgError if G + reg I is not positive definite."""
        if not self.reg_weight > 0:
            raise NotImplementedError(f'EASE needs reg > 0 so that X^T X + reg I is positive definite (the inverse does not '
                                      f'pivot); got reg = {self.reg_weight}')
        u = np.asarray(train_set[self.uid_name].values)
        i = np.asarray(train_set[self.iid_name].values)
        v = np.array(train_set[self.inter_name].values, dtype=np.float64)
        # scipy's coo checks (csr_matrix((values, (u, i)), shape)), before anything reaches the device
        for ids, hi, what in ((u, self.user_num, 'row'), (i, self.item_num, 'column')):
            if len(ids) and ids.max() >= hi:
                raise ValueError(f'{what} index exceeds matrix dimensions')
            if len(ids) and ids.min() < 0:
                raise ValueError(f'negative {what} index found')
        d_u = torch.from_numpy(u.astype(np.int32)).to(self.device)
        d_i = torch.from_numpy(i.astype(np.int32)).to(self.device)
        d_v = torch.from_numpy(np.ascontiguousarray(v)).to(self.device)
        self.item_similarity = None                      # free the previous B before the next n x n allocation
        X = ops.ease_csr(d_u, d_i, d_v, self.user_num, self.item_num)
        ws = ops.ease_workspace(X)
        B = ops.ease_gram(X, float(self.reg_weight), ws)
        ops.ease_inverse(B, ws)
        ops.ease_weights(B, ws)
        del ws
        self._X, self._csr_host = X, None
        self.item_similarity = B

    @property
    def interaction_matrix(self):
        """X as the reference keeps it: scipy csr_matrix float32 [U, I] (built on first use)."""
        if self._csr_host is None and self._X is not None:
            X = self._X
            self._csr_host = sp.csr_matrix((X.val.cpu().numpy(), X.col.cpu().numpy(), X.row_ptr.cpu().numpy()),
                                           shape=(self.user_num, self.item_num))
        return self._csr_host

    # ------------------------------------------------------------------ scoring
    def predict(self, u, i):
        """-> numpy.float64: x_u . B[:, i] (EASERecommender.py:49-50)."""
        us, its = self._ids((u,), (i,))
        return np.float64(ops.ease_predict(self.item_similarity, self._X, us, its).item())

    def rank(self, test_loader):
        """-> int64 ndarray [n_test_users, topk] of candidate ids by s_c = sum_i x_ui B[c, i] (EASERecommender.py:53-70)."""
        ins = self._rank_inputs(test_loader)
        if ins is None:
            return None
        users, cands, k = ins
        return ops.ease_rank(self.item_similarity, self._X, torch.from_numpy(users).to(self.device),
                             torch.from_numpy(cands).to(self.device), k).cpu().numpy()

    def full_rank(self, u):
        """-> int64 ndarray [1, topk] of the top items by x_u B; no masking of train items (EASERecommender.py:72-74)."""
        users = self._ids((u,))[0]
        return ops.ease_full_rank(self.item_similarity, self._X, users, min(self.topk, self.item_num)).cpu().numpy()

    def _ids(self, users, items=None):
        if self.item_similarity is None:
            raise RuntimeError('EASE: fit() must run before scoring')
        cols, bounds, names = [users], [self.user_num], ['user']
        if items is not None:
            cols, bounds, names = cols + [items], bounds + [self.item_num], names + ['item']
        self._check_ids(cols, bounds, names)
        return [torch.as_tensor(np.asarray(c, dtype=np.int64)).reshape(-1).to(self.device) for c in cols]
