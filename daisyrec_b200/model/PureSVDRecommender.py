"""PureSVD on the GPU path, with the reference's class name, config keys and methods (daisy/model/PureSVDRecommender.py).

fit(train_set) has no training loop: the reference runs sklearn's randomized_svd(X, factors, random_state=2019) on the host.
Here Omega is drawn on the host from the same RandomState (bit-exact with sklearn) and everything else runs on the device in
fp64 (csrc/puresvd.cu): the power rounds as SpMMs over X and X^T, every normaliser shifted CholeskyQR3 (the same subspace as
sklearn's LU / QR), the projected SVD by one-sided Jacobi, and sklearn's sign rule.  ``user_vec`` [U, k] and ``item_vec``
[I, k] are device fp64 tensors.

    fit        -> drb_csr_build + drb_skipgram_group + drb_puresvd_csr, drb_puresvd_spmm / orth / small_svd / factors
    rank       -> drb_puresvd_scores + drb_itemknn_topk: (score descending, candidate position ascending)
    full_rank  -> the same over every item, no masking of train items        predict -> drb_puresvd_scores

Users and items without train rows get exactly zero factor rows (a zero row of X stays zero through every product and row
normalisation); the reference's cold users carry LAPACK noise of about 1e-16 instead, so its order of their candidates is not
reproducible.  Here their rank is the candidate order.
"""
import numpy as np
import torch

from .. import ops
from .AbstractRecommender import DeviceRecommender

SEED = 2019                  # PureSVDRecommender.py: randomized_svd(..., random_state=2019)
OVERSAMPLES = 10             # sklearn's n_oversamples default
MAX_L = 1024                 # drb_puresvd_small_svd: one CTA of 1024 threads


class PureSVD(DeviceRecommender):
    MULTI_GPU = '{} runs on a single GPU'

    def __init__(self, config):
        """Same keys as the reference: user_num, item_num, factors, topk (+ gpu, logger)."""
        super().__init__(config)
        self.user_num = config['user_num']
        self.item_num = config['item_num']
        self.factors = config['factors']
        self.topk = config['topk']
        self.user_vec = None
        self.item_vec = None
        self.sigma = None

    # ------------------------------------------------------------------ fit
    def fit(self, train_set):
        """randomized_svd on the device.  numpy.linalg.LinAlgError if a panel is numerically rank deficient (rank(X) below
        factors + 10)."""
        U, I, k = int(self.user_num), int(self.item_num), int(self.factors)
        n, l = min(U, I), k + OVERSAMPLES
        if l > n:
            raise NotImplementedError(f'PureSVD needs factors + {OVERSAMPLES} <= min(user_num, item_num) = {n}; got factors = {k} '
                                      f'(sklearn returns fewer components there, which is not built)')
        if l > MAX_L:
            raise NotImplementedError(f'PureSVD supports factors + {OVERSAMPLES} <= {MAX_L} (the one-CTA Jacobi SVD); got '
                                      f'factors = {k}')
        self.logger.info('Computing SVD decomposition...')
        u = np.asarray(train_set['user'].values)
        i = np.asarray(train_set['item'].values)
        v = np.array(train_set['rating'].values, dtype=np.float64)
        # scipy's coo checks (csr_matrix((values, (u, i)), shape)), before anything reaches the device
        for ids, hi, what in ((u, U, 'row'), (i, I, 'column')):
            if len(ids) and ids.max() >= hi:
                raise ValueError(f'{what} index exceeds matrix dimensions')
            if len(ids) and ids.min() < 0:
                raise ValueError(f'negative {what} index found')
        transposed = U < I
        n_iter = 7 if k < 0.1 * n else 4
        omega = np.random.RandomState(SEED).normal(size=(n, l))
        d = lambda a, t: torch.from_numpy(np.ascontiguousarray(a, t)).to(self.device)
        self.user_vec = self.item_vec = self.sigma = None
        X = ops.puresvd_csr(d(u, np.int32), d(i, np.int32), d(v, np.float64), U, I)
        self.user_vec, self.item_vec, self.sigma = ops.puresvd_fit(X, omega, k, n_iter, transposed)
        self.logger.info('Done!')

    # ------------------------------------------------------------------ scoring
    def predict(self, u, i):
        """-> numpy.float64: user_vec[u] . item_vec[i]."""
        us, its = self._ids((u,), (i,))
        return np.float64(ops.puresvd_predict(self.user_vec, self.item_vec, us, its).item())

    def rank(self, test_loader):
        """-> int64 ndarray [n_test_users, topk] of candidate ids by (score descending, candidate position ascending)."""
        ins = self._rank_inputs(test_loader)
        if ins is None:
            return None
        users, cands, k = ins
        return ops.puresvd_rank(self.user_vec, self.item_vec, torch.from_numpy(users).to(self.device),
                                torch.from_numpy(cands).to(self.device), k).cpu().numpy()

    def full_rank(self, u):
        """-> int64 ndarray [topk] of the top items by user_vec[u] . item_vec^T; no masking of train items."""
        users = self._ids((u,))[0]
        return ops.puresvd_full_rank(self.user_vec, self.item_vec, users, min(self.topk, self.item_num)).cpu().numpy()[0]

    def _ids(self, users, items=None):
        if self.user_vec is None:
            raise RuntimeError('PureSVD: fit() must run before scoring')
        cols, bounds, names = [users], [self.user_num], ['user']
        if items is not None:
            cols, bounds, names = cols + [items], bounds + [self.item_num], names + ['item']
        self._check_ids(cols, bounds, names)
        return [torch.as_tensor(np.asarray(c, dtype=np.int64)).reshape(-1).to(self.device) for c in cols]
