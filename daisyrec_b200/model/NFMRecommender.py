"""NFM + BPR on the GPU path, with the reference's class name, config keys and methods
(daisy/model/NFMRecommender.py:14-209).

Factor tables ``embed_user.weight`` / ``embed_item.weight``, the first-order terms in one packed vector (``u_bias.weight``,
``i_bias.weight``, ``bias_`` are views of it), the network (FM_layers' BatchNorm, the hidden Linear / BatchNorm layers and
``prediction.weight``) in one flat fp32 block ``net`` in module-registration order, the BatchNorm running statistics in
``running`` (mean, var per BatchNorm).  Training goes through ``drb_nfm_bpr_train_steps``; rank / full_rank / predict score
in eval mode (running statistics) through ``drb_nfm_scores`` + ``drb_topk_from_scores``.

Dropout (``config['dropout']``, reference default 0.5, :67,:88) is active in train mode; eval-mode scoring is mask-free.  Where
the masks come from (``dropout_engine``):
- ``'auto'`` (default) / ``'torch'``: the host draws exactly the masks torch's Dropout modules would -- ``bernoulli_(1 - p)`` on
  the global CPU generator, forward(user, pos) first (FM_layers' Dropout, then the one behind each activation), then
  forward(user, neg) -- and uploads them as bytes with the batch, so a step equals the reference's and the global RNG ends where
  the reference's does.  That is a parity mechanism (one byte per activation and step through the host).
- ``'philox'``: the kernels draw the masks from Philox (same distribution, another stream), keyed by a seed -- one int64 drawn
  from torch's global generator the first time a fit needs it -- and the global step; the pos and neg calls draw independent
  masks and the backward regenerates them.  The throughput setting.

Two reference behaviours are NOT mirrored because they are failures, not results: with ``dropout = 0`` today's torch makes
the reference's own ``backward()`` raise (the in-place ``fm += ...`` of :120 aliases the activation output), and
``predict()`` with ``batch_norm`` feeds a 1-D row to BatchNorm1d, which rejects it.  Both work here.
"""
import numpy as np
import torch

from .. import ops
from .AbstractRecommender import GeneralRecommender, _Table, _init_table, _INIT, packed_bias, ragged_split


class NFM(GeneralRecommender):
    DEFAULT_INIT = 'xavier_normal'
    PARAMS = ('embed_user.weight', 'embed_item.weight', 'u_bias.weight', 'i_bias.weight', 'bias_', 'net')
    BUFFERS = ('running',)
    STRICT_STATE = False
    SCRATCH_KEY = 'nfm_scratch_rows'

    def __init__(self, config):
        super().__init__(config)
        self.act_function = config['act_function']
        self.num_layers = config['num_layers']
        self.batch_norm = bool(config['batch_norm'])
        self.dropout = float(config['dropout'] or 0.0)
        if not 0.0 <= self.dropout < 1.0:
            raise ValueError(f"dropout probability has to be in [0, 1), but got {self.dropout}")
        self.dropout_engine = str(config.get('dropout_engine', 'auto')).lower()
        if self.dropout_engine not in ('auto', 'torch', 'philox'):
            raise ValueError(f"dropout_engine must be 'auto', 'torch' or 'philox', got {self.dropout_engine!r}")
        self._philox_seed = None
        if self.act_function not in ops.NFM_ACT:
            raise NotImplementedError(f"act_function={self.act_function!r}: expected one of {sorted(ops.NFM_ACT)}")
        U, I, F, Ln = self.user_num, self.item_num, self.factors, self.num_layers

        # reference RNG stream (:55-108): constructors in registration order, then _init_weight
        import torch.nn as nn
        wu, wi = _init_table(U, F, None), _init_table(I, F, None)
        _init_table(U, 1, None); _init_table(I, 1, None)                 # u_bias / i_bias constructors (zeroed by _init_weight)
        linears = [nn.Linear(F, F) for _ in range(Ln)]                   # BatchNorm1d / Dropout constructors draw nothing
        prediction = nn.Linear(F, 1, bias=False)
        init = _INIT[self.initializer]
        with torch.no_grad():
            init(wu)
            init(wi)
            if Ln > 0:
                for lin in linears:
                    init(lin.weight)                                     # biases keep nn.Linear's own draw (:101-104)
                init(prediction.weight)
            else:
                prediction.weight.fill_(1.0)
            parts = []
            one, zero = torch.ones(F), torch.zeros(F)
            if self.batch_norm:
                parts += [one, zero]
            for lin in linears:
                parts += [lin.weight.reshape(-1), lin.bias.reshape(-1)]
                if self.batch_norm:
                    parts += [one, zero]
            parts.append(prediction.weight.reshape(-1))
            net = torch.cat(parts).contiguous()
        assert net.numel() == ops.nfm_param_count(F, Ln, self.batch_norm)
        self.embed_user = _Table(wu.to(self.device))
        self.embed_item = _Table(wi.to(self.device))
        self.bias, self.u_bias, self.i_bias, self.bias_ = packed_bias(U, I, self.device)
        self.net = net.to(self.device)
        n_bn = (1 + Ln) if self.batch_norm else 0
        run = torch.zeros(n_bn * 2 * F, dtype=torch.float32)
        for k in range(n_bn):
            run[k * 2 * F + F:(k + 1) * 2 * F] = 1.0                     # running_var starts at 1
        self.running = run.to(self.device)
        td = str(config.get('tower_dtype', 'fp32')).lower()
        if td not in ('fp32', 'bf16'):
            raise ValueError(f"tower_dtype must be 'fp32' or 'bf16', got {td!r}")
        self._tower_dtype = 1 if td == 'bf16' else 0
        self._act = ops.NFM_ACT[self.act_function]

    def _workspace(self, opt, rows):
        return ops.NfmWorkspace(self.user_num, self.item_num, self.factors, self.num_layers, self.batch_norm, opt, max(rows, 2),
                                self.device)

    def _begin_fit(self, opt):
        self._philox_seed = None                                         # drawn lazily: a fit without device masks draws nothing
        super()._begin_fit(opt)

    def _drop_seed(self):
        if self._philox_seed is None:
            self._philox_seed = int(torch.empty((), dtype=torch.int64).random_().item())
        return self._philox_seed

    def _host_keep(self, rows_per_step):
        """The masks nn.Dropout would draw for steps of rows_per_step[k] triples, drawn by torch on the global CPU generator in
        the reference's order -> uint8 CUDA tensor [step][forward call][site][rows][F] (drb_nfm_bpr_train_steps)."""
        F, sites, keep = self.factors, 1 + self.num_layers, 1.0 - self.dropout
        parts = []
        for B in rows_per_step:
            for _side in (0, 1):                                          # forward(user, pos) draws first, then forward(user, neg)
                for _site in range(sites):
                    parts.append(torch.empty(B, F, dtype=torch.float32).bernoulli_(keep).to(torch.uint8).reshape(-1))
        return torch.cat(parts).to(self.device)

    def _launch(self, bu, bi, bj, batch, first, n_steps, apply=True):
        """n_steps steps; in train mode with dropout > 0 the masks of every step are drawn first (in step order)."""
        kw = dict(adam_step0=self._opt_steps, tower_dtype=self._tower_dtype, apply=apply)
        args = (self.embed_user.weight, self.embed_item.weight, self.bias, self.net, self.running, self._ws, self._act)
        if not (self.training and self.dropout > 0.0):
            return ops.nfm_bpr_train_steps(*args, bu, bi, bj, batch, first, n_steps, self._hp, **kw)
        if self.dropout_engine == 'philox':
            return ops.nfm_bpr_train_steps_philox(*args, bu, bi, bj, batch, first, n_steps, self._hp, dropout=self.dropout,
                                                  seed=self._drop_seed(), **kw)
        per_step = 2 * (1 + self.num_layers) * batch * self.factors
        chunk = max(1, (64 << 20) // per_step)                           # at most 64 MB of masks per call
        out, s = [], first
        while s < first + n_steps:
            k = min(chunk, first + n_steps - s)
            full, last = ragged_split(bu.numel(), batch, s, k)
            if full > 0:
                out.append(ops.nfm_bpr_train_steps(*args, bu, bi, bj, batch, s, full, self._hp, dropout=self.dropout,
                                                   keep=self._host_keep([batch] * full),
                                                   **dict(kw, adam_step0=self._opt_steps + (s - first))))
            if last:
                base = (s + full) * batch
                out.append(ops.nfm_bpr_train_steps(*args, bu[base:], bi[base:], bj[base:], last, 0, 1, self._hp, dropout=self.dropout,
                                                   keep=self._host_keep([last]),
                                                   **dict(kw, adam_step0=self._opt_steps + (s + full - first))))
            s += k
        return torch.cat(out)

    # ------------------------------------------------------------------ reference surface
    def _scores(self, u, i):
        self._ensure(2)
        return ops.nfm_scores(self.embed_user.weight, self.embed_item.weight, self.bias, self.net, self.running, self._ws,
                              self._act, u, i, self._tower_dtype)

    def _pair_scores(self, user, item):
        """NFMRecommender.py:110-123 in eval mode (running statistics) for index tensors."""
        return self._scores(*self._pair_ids(user, item))

    def rank(self, test_loader):
        ins = self._rank_inputs(test_loader)
        if ins is None:
            return np.zeros((0,), np.float32)
        users, cands, k = ins
        n, C = cands.shape
        d_cands = torch.from_numpy(cands).to(self.device)
        u_rep = torch.from_numpy(np.repeat(users, C).astype(np.int32)).to(self.device)
        scores = self._scores(u_rep, d_cands.reshape(-1).to(torch.int32).contiguous()).view(n, C).contiguous()
        return ops.topk_from_scores(scores, d_cands, k).cpu().numpy()

    def full_rank(self, u):
        self._check_ids(([int(u)],), (self.user_num,), ('user',))
        items = torch.arange(self.item_num, dtype=torch.int32, device=self.device)
        users = torch.full((self.item_num,), int(u), dtype=torch.int32, device=self.device)
        scores = self._scores(users, items).view(1, -1).contiguous()
        return ops.topk_from_scores(scores, None, min(self.topk, self.item_num))[0].cpu().numpy()
