"""SLiM on the GPU path, with the reference's class name, config keys and methods (daisy/model/SLiMRecommender.py:27-157).

fit(train_set) solves every item's ElasticNet at once on the device (csrc/slim.cu on csrc/ease.cu's CSR and Gram matrix):

    fit        -> drb_csr_build + drb_ease_csr, drb_ease_gram (reg 0),
                  per panel of items drb_slim_live + drb_slim_solve + drb_slim_select
    rank / full_rank / predict -> drb_itemknn_scores (+ drb_itemknn_topk), as ItemKNNCF

Item j's fit is min_{w >= 0, w_j = 0} 1/2 w^T G w - G[:, j]^T w + l1 sum(w) + 1/2 l2 |w|^2 with G = X^T X,
l1 = alpha elastic U, l2 = alpha (1 - elastic) U: what sklearn's ElasticNet(positive=True, fit_intercept=False) minimises,
times U.  l2 > 0 makes it strongly convex, so the optimum is unique; the reference visits coordinates in a random order drawn
from numpy's global RandomState, so its iterates cannot be reproduced, but its optimum can.  The stopping rule is sklearn's
(formulation-A duality gap <= tol G_jj, checked when the sweep's relative step is below tol), so each column is certified to
lie within sqrt(2 gap / l2) of the optimum.

A_tilde = X W is NOT materialised: entries are summed on demand in fp64 over ascending neighbour ids, the order scipy's csr
product adds in.  Among equal coefficients at the topk cut the lower item ids are kept (the reference leaves that to
argpartition).
"""
import numpy as np
import torch

from .. import ops
from .AbstractRecommender import NeighbourScorer

RAND_R_MAX = 2147483647      # sklearn's cd_fast draws rng.randint(0, RAND_R_MAX) once per ElasticNet.fit


class SLiM(NeighbourScorer):
    MULTI_GPU = '{} runs on a single GPU'

    def __init__(self, config):
        """Same keys as the reference (SLiMRecommender.py:41-52): alpha, elastic, topk, user_num, item_num (+ gpu, logger).
        Optional: slim_tol (1e-4) and slim_max_iter (100), sklearn's tol and max_iter as the reference fixes them."""
        super().__init__(config)
        self.alpha = config['alpha']
        self.elastic = config['elastic']
        self.item_num = config['item_num']
        self.user_num = config['user_num']
        self.topk = config['topk']
        self.tol = float(config.get('slim_tol', 1e-4))
        self.max_iter = int(config.get('slim_max_iter', 100))
        self._X = self._W = self._w_host = None
        self.sweeps = self.gaps = self.converged = None
        self.logger.info(f'user num: {self.user_num}, item num: {self.item_num}')

    # ------------------------------------------------------------------ fit
    def fit(self, train_set, verbose=True):
        """SLiMRecommender.py:59-124 on the device.  MemoryError when the fp64 [I, I] Gram matrix and one panel of solver
        state do not fit in the free device memory."""
        alpha, elastic, topk = float(self.alpha), float(self.elastic), int(self.topk)
        if not alpha > 0:
            raise NotImplementedError(f'SLiM needs alpha > 0 on the GPU path; got {self.alpha}')
        if not 0 < elastic < 1:
            raise NotImplementedError(f'SLiM needs elastic in (0, 1) on the GPU path (l2 > 0 makes the optimum unique); '
                                      f'got {self.elastic}')
        if not 1 <= topk <= 1024:
            raise NotImplementedError(f'SLiM keeps 1 to 1024 coefficients per item on the GPU path; got topk = {self.topk}')
        u = np.asarray(train_set['user'].values)
        i = np.asarray(train_set['item'].values)
        v = np.array(train_set['rating'].values, dtype=np.float64)
        self._check_ids((u, i), (self.user_num, self.item_num), ('user', 'item'))
        n, U = self.item_num, self.user_num
        self._X = self._W = self._w_host = None             # free the previous fit before the n x n allocation
        torch.cuda.empty_cache()
        lib = ops.L.lib()
        per_target = lib.drb_slim_workspace_bytes(n, 1) - 8 * n
        free = torch.cuda.mem_get_info(self.device)[0]
        base = 8 * n * n + 24 * len(u) + 8 * U + (8 * topk + 64) * n
        need = base + max(lib.drb_ease_workspace_bytes(U, n, -1), 8 * n + per_target * min(n, 64))
        if need > free:
            raise MemoryError(f'SLiM.fit needs {need} bytes of device memory for {n} items (the dense fp64 Gram matrix alone is '
                              f'{8 * n * n}); {free} bytes are free')
        d = lambda a, t: torch.from_numpy(np.ascontiguousarray(a, t)).to(self.device)
        X = ops.ease_csr(d(u, np.int32), d(i, np.int32), d(v, np.float64), U, n)
        ws = ops.ease_workspace(X)
        G = ops.ease_gram(X, 0.0, ws)
        del ws
        torch.cuda.empty_cache()
        all_live = bool(X.val.numel()) and bool((X.val < 0).any())
        l1, l2 = alpha * elastic * U, alpha * (1.0 - elastic) * U
        free = torch.cuda.mem_get_info(self.device)[0]
        panel = int(min(n, (free - (8 * topk + 64) * n - 8 * n - (256 << 20)) // per_target))
        if panel < min(n, 64):
            raise MemoryError(f'SLiM.fit: {free} bytes are free next to the {8 * n * n}-byte Gram matrix, less than one panel '
                              f'of {min(n, 64)} items needs ({per_target} bytes per item)')
        W = None
        sweeps, gaps, conv = [], [], []
        for b in range(0, n, panel):
            P = ops.slim_solve(G, l1, l2, self.tol, self.max_iter, b, min(panel, n - b), all_live)
            W = ops.slim_select(P, topk, W)
            sweeps.append(P.sweeps.cpu()), gaps.append(P.gap.cpu()), conv.append(P.conv.cpu())
            del P
        del G
        self.sweeps = torch.cat(sweeps).numpy()
        self.gaps = torch.cat(gaps).numpy() / U                   # sklearn's dual_gap_
        self.converged = torch.cat(conv).numpy().astype(bool)
        stopped = int((~self.converged).sum())
        if stopped:
            self.logger.warning(f'SLiM: {stopped} of {n} item columns stopped at max_iter = {self.max_iter} before the duality '
                                f'gap reached tol')
        if verbose:
            self.logger.info(f'SLIM-ElasticNet-Recommender: Processed {n} items, {int(self.sweeps.sum())} sweeps')
        self._X, self._W = X, W
        # the reference's ElasticNet.fit draws one seed per item from numpy's global RandomState (selection='random')
        np.random.randint(0, RAND_R_MAX, size=n)

    @property
    def w_sparse(self):
        """W as the reference builds it: scipy csr_matrix float32 [I, I], column c holding item c's coefficients (built on
        first use)."""
        if self._w_host is None and self._W is not None:
            self._w_host = self._neighbour_csc().tocsr()
        return self._w_host

    # ------------------------------------------------------------------ scoring
    def predict(self, u, i):
        """-> numpy.float64: A_tilde[u, i] (SLiMRecommender.py:126-127)."""
        return self._predict_score(u, i)

    def rank(self, test_loader):
        """-> int64 ndarray [n_test_users, topk] of candidate ids by A_tilde[u, c], ties by candidate position
        (SLiMRecommender.py:129-141); None for an empty loader."""
        return super().rank(test_loader)

    def full_rank(self, u):
        """-> int64 ndarray [topk] of the top items of user u; no masking of train items (SLiMRecommender.py:143-146)."""
        return super().full_rank(u)
