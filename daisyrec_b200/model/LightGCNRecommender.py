"""LightGCN + BPR on the GPU path, with the reference's class name, config keys and methods
(daisy/model/LightGCNRecommender.py:23-211).

The ego table E0 = cat(embed_user.weight, embed_item.weight) is one contiguous device tensor
(``embed_user.weight`` / ``embed_item.weight`` are views of it); the normalised adjacency is built once
on the host exactly as ``get_norm_adj_mat`` does (:73-107, values bit-identical) and lives on the device as
segmented CSR.  Every step runs L forward + L backward sparse products and the fused BPR / Adam kernels
through ``drb_lgcn_bpr_train_steps``; rank / full_rank / predict score with the cached propagated
tables (``restore_user_e`` / ``restore_item_e``, :64-65) through the MF rank kernels.
"""
import numpy as np
import torch

from .. import ops
from .AbstractRecommender import GeneralRecommender, _Table, _init_table, _INIT


class LightGCN(GeneralRecommender):
    DEFAULT_OPTIMIZER, DEFAULT_INIT = 'adam', 'xavier_uniform'

    def __init__(self, config):
        super().__init__(config)
        self.interaction_matrix = config['inter_matrix']            # scipy COO from utils.get_inter_matrix
        self.num_layers = config['num_layers']

        # reference init stream: two nn.Embedding constructors, then apply(_init_weight) (LightGCNRecommender.py:53-68)
        wu = _init_table(self.user_num, self.factors, None)
        wi = _init_table(self.item_num, self.factors, None)
        _INIT[self.initializer](wu)
        _INIT[self.initializer](wi)
        self.E0 = torch.cat([wu, wi]).contiguous().to(self.device)
        self.embed_user = _Table(self.E0[:self.user_num])
        self.embed_item = _Table(self.E0[self.user_num:])
        self.restore_user_e = None
        self.restore_item_e = None

        m = self.interaction_matrix
        # optional GPU-path key 'adj_builder': 'host' (default; numpy restatement of get_norm_adj_mat, values bit-identical to
        # scipy's) | 'device' (sorted CSR + transpose + D^-1/2 A D^-1/2 built by csr.cu; 1/sqrt instead of pow: fp32
        # values equal except on rare rounding ties)
        if str(config.get('adj_builder', 'host')) == 'device':
            row_ptr, col, val = ops.lgcn_build_adj(torch.from_numpy(np.ascontiguousarray(m.row, np.int32)).to(self.device),
                                                   torch.from_numpy(np.ascontiguousarray(m.col, np.int32)).to(self.device),
                                                   self.user_num, self.item_num)
        else:
            row_ptr, col, val = ops.lgcn_norm_adj(np.asarray(m.row), np.asarray(m.col), self.user_num, self.item_num)
        self.graph = ops.LgcnGraph(row_ptr, col, val, self.device)

    def _workspace(self, opt, rows=None):
        return ops.LgcnWorkspace(self.user_num, self.item_num, self.factors, opt, self.device)

    def _launch(self, bu, bi, bj, batch, first, n_steps, apply=True):
        self._drop_cache()                                           # LightGCNRecommender.py:133-134
        return ops.lgcn_bpr_train_steps(self.E0, self._ws, self.graph, self.num_layers, bu, bi, bj, batch, first, n_steps,
                                        self._hp, adam_step0=self._opt_steps if apply else 0, apply=apply)

    # ------------------------------------------------------------------ reference surface
    def forward(self):
        """LightGCNRecommender.py:117-129 -> (user_embedding, item_embedding) after propagation + layer mean."""
        self._ensure()
        Em = ops.lgcn_propagate(self.E0, self._ws, self.graph, self.num_layers)
        return Em[:self.user_num], Em[self.user_num:]

    def _drop_cache(self):
        self.restore_user_e = self.restore_item_e = None

    def _dot_tables(self):
        """rank / full_rank / predict score the cached propagated tables with MF's kernels."""
        if self.restore_user_e is None or self.restore_item_e is None:
            self.restore_user_e, self.restore_item_e = self.forward()
        return self.restore_user_e, self.restore_item_e
