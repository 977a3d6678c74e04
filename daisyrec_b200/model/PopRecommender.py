"""MostPop on the GPU path, with the reference's class name, config keys, attributes and methods (daisy/model/PopRecommender.py).

    fit                -> drb_mostpop_fit (value_counts by integer atomics, item_score = cnt / (1 + cnt) in fp64), and the
                          full_rank order once: drb_itemknn_topk over every item
    rank               -> drb_mostpop_gather + drb_itemknn_topk
    predict, full_rank -> the host copies fit keeps

Ties.  Popularity scores tie constantly, and the reference orders them with torch.argsort (rank) and np.argsort (full_rank),
neither of them stable, so its order inside a group of equal scores is not reproducible.  This path's rule is (score
descending, candidate position ascending) for rank and (score descending, item id ascending) for full_rank.
"""
import numpy as np
import torch

from .. import ops
from .AbstractRecommender import DeviceRecommender


class MostPop(DeviceRecommender):
    MULTI_GPU = '{} runs on a single GPU'

    def __init__(self, config):
        """Same keys as the reference (PopRecommender.py:17-27): item_num, topk, IID_NAME (+ gpu, logger)."""
        super().__init__(config)
        self.item_num = config['item_num']
        self.item_cnt_ref = np.zeros(self.item_num)
        self.topk = config['topk']
        self.cnt_col = config['IID_NAME']
        self._score = self._order = None

    def fit(self, train_set):
        """PopRecommender.py:29-33: every row of the IID_NAME column counted, duplicates included.  IndexError for an id
        outside [0, item_num): the reference raises for ids >= item_num and wraps negative ones silently; this path refuses
        both.  Each fit counts from zero: the reference assigns the new counts into its existing item_cnt_ref, so after a
        second fit its items absent from the new train set keep their old counts; here they count 0."""
        ids = np.asarray(train_set[self.cnt_col].values)
        if ids.dtype.kind not in 'iu':
            raise IndexError(f'{self.cnt_col} ids must be integers; got dtype {ids.dtype}')
        d_ids = torch.from_numpy(np.array(ids, dtype=np.int64)).to(self.device)
        cnt, score = ops.mostpop_fit(d_ids, self.item_num)
        self._score = score
        self._order = ops.mostpop_order(score, min(self.topk, self.item_num)).cpu().numpy()
        self.item_cnt_ref = cnt.cpu().numpy()
        self.item_score = score.cpu().numpy()

    def predict(self, u, i):
        """-> item_score[i] (PopRecommender.py:35-36)."""
        return self.item_score[i]

    def rank(self, test_loader):
        """-> float32 ndarray [n_test_users, min(topk, C)] of candidate ids by (score descending, candidate position ascending),
        rows in loader order; the ids are float32 because the reference concatenates onto torch.tensor([])
        (PopRecommender.py:38-50)."""
        if self._score is None:
            raise RuntimeError('MostPop: fit() must run before scoring')
        cs = [torch.as_tensor(c).to(torch.int64).reshape(len(us), -1) for us, c in test_loader]
        cs = [c for c in cs if c.numel()]
        if not cs:
            return np.zeros((0,), np.float32)
        cands = torch.cat(cs)
        self._check_ids((cands,), (self.item_num,), ('candidate item',))
        cands = cands.to(self.device).contiguous()
        out = ops.mostpop_rank(self._score, cands, min(self.topk, cands.shape[1]))
        return out.to(torch.float32).cpu().numpy()

    def full_rank(self, u):
        """-> int64 ndarray [min(topk, item_num)]: the same items for every user (PopRecommender.py:52-53)."""
        if self._order is None:
            raise RuntimeError('MostPop: fit() must run before scoring')
        return self._order.copy()
