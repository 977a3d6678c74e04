"""Item2Vec on the GPU path, with the reference's class name, config keys and methods
(daisy/model/Item2VecRecommender.py:16-107).

One tied item table (``shared_embedding.weight``) trained on the skip-gram rows of SkipGramNegativeSampler with
BCEWithLogitsLoss(sum) and no regulariser; after every fit() the user table is rebuilt as the sum of each train user's
item rows.  Ranking is MF's with P = ``user_embedding.weight`` and Q = ``shared_embedding.weight``.

    fit        -> drb_gather_triples + drb_i2v_train_steps (one persistent launch per epoch) + drb_i2v_user_embedding
    calc_loss  -> drb_i2v_train_steps (apply = 0)          train_step -> drb_i2v_train_steps (one batch)
    rank / full_rank / predict -> drb_mf_rank / drb_mf_full_rank / drb_mf_predict
"""
import numpy as np
import torch

from .. import ops
from ..utils.sampler import csr_from_ur
from .AbstractRecommender import GeneralRecommender, _Table, _init_table, _INIT
from .MFRecommender import MF


class Item2Vec(GeneralRecommender):
    SUPPORTED_LOSSES = ('CL',)
    DEFAULT_OPTIMIZER = 'adam'
    LOSS_TYPE = 'CL'
    PARAMS = ('user_embedding.weight', 'shared_embedding.weight')

    def __init__(self, config):
        """Same keys as the reference (Item2VecRecommender.py:18-46): user_num, item_num, factors, train_ur, lr, epochs,
        optimizer, init_method, early_stop, topk (+ gpu, logger).  loss_type is always CL."""
        super().__init__(config)
        self.ur = config['train_ur']
        # the reference's CPU RNG consumption: nn.Embedding(user_num), nn.Embedding(item_num), then apply(_init_weight)
        wu = _init_table(self.user_num, self.factors, None)
        wi = _init_table(self.item_num, self.factors, None)
        _INIT[self.initializer](wu)
        _INIT[self.initializer](wi)
        self.user_embedding = _Table(wu.to(self.device))
        self.shared_embedding = _Table(wi.to(self.device))
        self._train_csr = config.get('train_csr', None)            # (row_ptr int64, col int32) to skip the dict walk
        self._csr_dev = None

    # MF's scoring with P = user_embedding, Q = shared_embedding (Item2VecRecommender.py:71-107 are MFRecommender.py:99-133)
    embed_user = property(lambda self: self.user_embedding)
    embed_item = property(lambda self: self.shared_embedding)
    _full_user_table = MF._full_user_table
    full_rank_users = MF.full_rank_users

    def _index_bounds(self):
        return (self.item_num, self.item_num, 1 << 62), ('target item', 'context item', 'label')

    def _workspace(self, opt, rows=None):
        return ops.I2VWorkspace(self.item_num, self.factors, opt, self.device)

    def _launch(self, bu, bi, bj, batch, first, n_steps, apply=True):
        return ops.i2v_train_steps(self.shared_embedding.weight, self._ws, bu, bi, bj, batch, first, n_steps, self._hp,
                                   adam_step0=self._opt_steps, apply=apply)

    # ------------------------------------------------------------------ reference surface
    def fit(self, train_loader):
        super().fit(train_loader)
        self.logger.info('Start building user embedding...')
        self.build_user_embedding()

    def build_user_embedding(self):
        """user_embedding[u] = shared_embedding[train_ur[u]].sum(0) for every user of train_ur (Item2VecRecommender.py:58-61);
        the other users keep their rows."""
        if self._csr_dev is None:
            row_ptr, col = self._train_csr if self._train_csr is not None else csr_from_ur(self.ur, self.user_num)
            self._csr_dev = (torch.from_numpy(np.ascontiguousarray(row_ptr, np.int64)).to(self.device),
                             torch.from_numpy(np.ascontiguousarray(col, np.int32)).to(self.device))
        ops.i2v_user_embedding(self.shared_embedding.weight, self._csr_dev[0], self._csr_dev[1], self.user_embedding.weight)

    def calc_loss(self, batch):
        """Item2VecRecommender.py:63-69: 0-d fp32 loss of one (target, context, label) batch; no update.  An empty batch
        launches nothing: its loss is 0."""
        if len(batch[0]) == 0:
            self._ensure()
            return torch.zeros((), dtype=torch.float32, device=self.device)
        return super().calc_loss(batch)

    def train_step(self, batch):
        if len(batch[0]) == 0:
            self._ensure()
            return 0.
        return super().train_step(batch)
