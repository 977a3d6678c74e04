"""NGCF + BPR on the GPU path, with the reference's class name, config keys and methods
(daisy/model/NGCFRecommender.py:61-252).

The ego table E0 = cat(embed_user.weight, embed_item.weight) is one contiguous device tensor; the BiGNN layers live in
one flat fp32 block (``gnn``: per layer W1, b1, W2, b2 in module-registration order); the normalised adjacency is
LightGCN's (``get_norm_adj_mat`` :125-146 is the same arithmetic) as segmented CSR on the device.  A step runs through
``drb_ngcf_bpr_train_steps`` (sparse products, GEMMs, the row-wise LeakyReLU / normalise kernels and the shared BPR /
optimiser phases); rank / full_rank / predict score the cached concatenated representation (``restore_user_e`` /
``restore_item_e``, :99-100) with the MF rank kernels.

Message dropout (``mess_dropout``, reference default 0.1): forward() builds ``nn.Dropout(mess_dropout)`` per layer (:164), a
module in training mode, so the reference drops on EVERY forward() -- the one behind rank() / full_rank() / predict() as well.
Node dropout (``node_dropout``, reference default 0): ``SparseDropout`` (:19-35) keeps every stored entry of the adjacency with
probability 1 - p and scales it by 1 / (1 - p), once per forward() and only in train mode (fit's steps, train_step, calc_loss
and forward() while ``model.training``; fit ends each epoch in eval mode, so rank() after fit drops messages but not edges).

Where the masks come from (``dropout_engine``):
- ``'auto'`` (default) / ``'torch'``: the host draws exactly the reference's message masks (one ``bernoulli_(1 - p)`` per layer
  over its [n, width] output, torch's global CPU generator) and uploads them as bytes; the kernels apply them between LeakyReLU
  and the row normalisation, forward and backward.  That is a parity mechanism (one byte per node and width through the host
  per forward).  ``node_dropout`` must be 0 here: host parity would need 2 * nnz host draws per forward.
- ``'philox'``: message and node masks are drawn inside the kernels from Philox (same distributions, another stream), keyed by
  a seed -- one int64 drawn from torch's global generator the first time a fit needs it -- and the model's forward counter,
  which advances once per forward(): once per training step and once per scoring forward, so the masks do not depend on
  ``steps_per_launch``.  The backward regenerates the message masks and multiplies by the transpose of the dropped adjacency
  through the CSR's mirror index (``LgcnGraph.edge_mirror``, built once when node dropout is on).
"""
import numpy as np
import torch

from .. import ops
from .AbstractRecommender import GeneralRecommender, _Table, _init_table, _INIT
from .LightGCNRecommender import LightGCN


class NGCF(GeneralRecommender):
    DEFAULT_OPTIMIZER, DEFAULT_INIT = 'adam', 'xavier_normal'
    PARAMS = ('embed_user.weight', 'embed_item.weight', 'gnn')

    def __init__(self, config):
        super().__init__(config)
        self.interaction_matrix = config['inter_matrix']            # scipy COO from utils.get_inter_matrix
        self.embedding_size = self.factors
        hidden = config['hidden_size_list'] if config.get('hidden_size_list') is not None else [64, 64, 64]
        self.hidden_size_list = [self.embedding_size] + list(hidden)
        self.node_dropout = config['node_dropout']
        self.message_dropout = config['mess_dropout']
        engine = str(config.get('dropout_engine', 'auto')).lower()
        if engine not in ('auto', 'torch', 'philox'):
            raise ValueError(f"dropout_engine must be 'auto', 'torch' or 'philox', got {engine!r}")
        self.dropout_engine = engine
        if engine == 'philox':
            self.node_dropout = float(self.node_dropout or 0.0)
            if not 0.0 <= self.node_dropout < 1.0:
                raise ValueError(f"node_dropout has to be in [0, 1), but got {self.node_dropout}")
        elif float(self.node_dropout or 0.0) != 0.0:
            raise NotImplementedError('NGCF on the GPU path runs node_dropout only with dropout_engine=\'philox\' (the reference '
                                      'draws its sparse dropout of the adjacency from the torch RNG)')
        self.message_dropout = float(self.message_dropout or 0.0)
        if not 0.0 <= self.message_dropout < 1.0:
            raise ValueError(f"dropout probability has to be in [0, 1), but got {self.message_dropout}")
        dims = self.hidden_size_list
        if any(int(d) < 1 or int(d) > 256 for d in dims):
            raise NotImplementedError('NGCF on the GPU path supports layer widths up to 256')

        # reference RNG stream (:95-116): two nn.Embedding constructors, per BiGNN layer two nn.Linear constructors, then
        # apply(_init_weight) over embed_user, embed_item and every (linear, interact_transform) pair
        import torch.nn as nn
        wu = _init_table(self.user_num, self.embedding_size, None)
        wi = _init_table(self.item_num, self.embedding_size, None)
        layers = [(nn.Linear(i, o), nn.Linear(i, o)) for i, o in zip(dims[:-1], dims[1:])]
        init = _INIT[self.initializer]
        with torch.no_grad():
            init(wu)
            init(wi)
            parts = []
            for lin, inter in layers:
                for mod in (lin, inter):
                    init(mod.weight)
                    mod.bias.zero_()
                parts += [lin.weight.reshape(-1), lin.bias.reshape(-1), inter.weight.reshape(-1), inter.bias.reshape(-1)]
            gnn = torch.cat(parts).contiguous()
        assert gnn.numel() == ops.ngcf_param_count(dims)
        self.E0 = torch.cat([wu, wi]).contiguous().to(self.device)
        self.embed_user = _Table(self.E0[:self.user_num])
        self.embed_item = _Table(self.E0[self.user_num:])
        self.gnn = gnn.to(self.device)
        self.restore_user_e = None
        self.restore_item_e = None
        m = self.interaction_matrix
        row_ptr, col, val = ops.lgcn_norm_adj(np.asarray(m.row), np.asarray(m.col), self.user_num, self.item_num)
        self.graph = ops.LgcnGraph(row_ptr, col, val, self.device)
        td = str(config.get('tower_dtype', 'fp32')).lower()
        if td not in ('fp32', 'bf16'):
            raise ValueError(f"tower_dtype must be 'fp32' or 'bf16', got {td!r}")
        self._tower_dtype = 1 if td == 'bf16' else 0
        self._forwards = 0                                           # forward() calls so far: the Philox masks' counter
        self._philox_seed = None

    def _workspace(self, opt, rows=None):
        return ops.NgcfWorkspace(self.user_num, self.item_num, self.hidden_size_list, opt, self.device)

    def _host_keep(self, n_forwards):
        """The masks nn.Dropout(mess_dropout) draws for n_forwards forward() calls: per call one bernoulli_ per layer over its
        [n, width] output on torch's global CPU generator -> uint8 CUDA tensor (None without message dropout)."""
        if self.message_dropout <= 0.0:
            return None
        n, keep = self.user_num + self.item_num, 1.0 - self.message_dropout
        parts = []
        for _ in range(n_forwards):
            for width in self.hidden_size_list[1:]:
                parts.append(torch.empty(n, int(width), dtype=torch.float32).bernoulli_(keep).to(torch.uint8).reshape(-1))
        return torch.cat(parts).to(self.device)

    def _begin_fit(self, opt):
        self._philox_seed = None                                     # drawn lazily: a fit without device masks draws nothing
        super()._begin_fit(opt)

    def _philox(self):
        """-> (seed, node dropout of this forward) when the masks come from the device, else None."""
        node = self.node_dropout if self.training else 0.0           # SparseDropout is the identity in eval mode (:30-31)
        if self.dropout_engine != 'philox' or (self.message_dropout <= 0.0 and node <= 0.0):
            return None
        if self._philox_seed is None:
            self._philox_seed = int(torch.empty((), dtype=torch.int64).random_().item())
        return self._philox_seed, node

    def _next_forwards(self, k):
        first = self._forwards
        self._forwards += k
        return first

    def _launch(self, bu, bi, bj, batch, first, n_steps, apply=True):
        self._drop_cache()                                           # NGCFRecommender.py:175-176
        ph = self._philox()
        if ph is not None:
            return ops.ngcf_bpr_train_steps_philox(self.E0, self.gnn, self._ws, self.graph, bu, bi, bj, batch, first, n_steps,
                                                   self._hp, adam_step0=self._opt_steps if apply else 0, apply=apply,
                                                   tower_dtype=self._tower_dtype, seed=ph[0],
                                                   forward0=self._next_forwards(1 if not apply else n_steps),
                                                   mess_dropout=self.message_dropout, node_dropout=ph[1])
        kw = dict(apply=apply, tower_dtype=self._tower_dtype, dropout=self.message_dropout)
        if self.message_dropout <= 0.0:
            return ops.ngcf_bpr_train_steps(self.E0, self.gnn, self._ws, self.graph, bu, bi, bj, batch, first, n_steps, self._hp,
                                            adam_step0=self._opt_steps if apply else 0, **kw)
        chunk = max(1, (64 << 20) // max(1, ops.ngcf_keep_bytes(self._ws)))   # masks of at most 64 MB per call, in step order
        out = []
        for s in range(first, first + n_steps, chunk):
            k = min(chunk, first + n_steps - s)
            out.append(ops.ngcf_bpr_train_steps(self.E0, self.gnn, self._ws, self.graph, bu, bi, bj, batch, s, k, self._hp,
                                                adam_step0=self._opt_steps + (s - first) if apply else 0,
                                                keep=self._host_keep(k), **kw))
        return torch.cat(out)

    # ------------------------------------------------------------------ reference surface
    def forward(self):
        """NGCFRecommender.py:157-172 -> (user_all_embeddings, item_all_embeddings): the concatenated layer outputs."""
        self._ensure()
        ph = self._philox()
        if ph is not None:
            rep = ops.ngcf_forward_philox(self.E0, self.gnn, self._ws, self.graph, self._tower_dtype, seed=ph[0],
                                          forward=self._next_forwards(1), mess_dropout=self.message_dropout, node_dropout=ph[1])
            return rep[:self.user_num], rep[self.user_num:]
        rep = ops.ngcf_forward(self.E0, self.gnn, self._ws, self.graph, self._tower_dtype, dropout=self.message_dropout,
                               keep=self._host_keep(1))              # the reference's forward() always drops (:164)
        return rep[:self.user_num], rep[self.user_num:]

    _drop_cache = LightGCN._drop_cache
    _dot_tables = LightGCN._dot_tables
