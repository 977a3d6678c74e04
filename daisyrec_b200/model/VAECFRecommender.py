"""Multi-VAE on the GPU path, with the reference's class name, config keys and methods (daisy/model/VAECFRecommender.py).

The network lives in one flat fp32 device block ``net`` in module order (csrc/vae.cu): per ``nn.Linear`` its weight, then its
bias, the first encoder weight stored item-major [I, hidden[0]].  ``state_dict()`` shows the reference's keys and shapes as views
of that block (``encoder.0.weight`` is the transposed view).  Training goes through ``drb_vae_train_steps``; rank / full_rank /
predict score in eval mode through ``drb_vae_scores`` + ``drb_topk_from_scores``.

Randomness in train mode (``dropout_engine``):
- ``'auto'`` / ``'torch'``: the host draws what the reference's forward() draws, on the global CPU generator and in its order:
  per step the dense [B, I] keep mask of F.dropout (``bernoulli_(1 - p)``, none when p = 0), then ``randn_like(std)``
  [B, latent_dim // 2].  The mask goes to the device bit-packed.  A step then equals the reference's, and the global RNG ends
  where the reference's fit leaves it.  The mask is B * I draws per step on the host.
- ``'philox'``: keep bits at the batch's nonzeros and the normals come from Philox on the device (same distributions, another
  stream): the throughput setting.
"""
import numpy as np
import torch

from .. import ops
from ..utils.sampler import fingerprint
from .AbstractRecommender import GeneralRecommender, _INIT, loader_plan, ragged_split


def _int_rows(data):
    return data.ndim == 1 and data.dtype.kind in 'iu'


class VAECF(GeneralRecommender):
    DEFAULT_OPTIMIZER = 'adam'
    DEFAULT_INIT = 'xavier_normal'
    LOSS_TYPE = 'VAE'
    SUPPORTED_LOSSES = ('VAE',)
    SCORE_ROWS = 1024                           # users per scoring pass

    def __init__(self, config):
        super().__init__(dict(config, factors=None))
        self.dropout = float(config['dropout'] or 0.0)
        if not 0.0 <= self.dropout < 1.0:
            raise ValueError(f"dropout probability has to be in [0, 1), but got {self.dropout}")
        self.layers = list(config['mlp_hidden_size']) if config['mlp_hidden_size'] is not None else [600]
        self.lat_dim = int(config['latent_dim'])
        if self.lat_dim < 2:
            raise ValueError(f"latent_dim must be >= 2, got {self.lat_dim}")
        self.anneal_cap = config['anneal_cap']
        self.total_anneal_steps = config['total_anneal_steps']
        self.update = 0
        engine = str(config.get('dropout_engine', 'auto')).lower()
        if engine not in ('auto', 'torch', 'philox'):
            raise ValueError(f"dropout_engine must be 'auto', 'torch' or 'philox', got {engine!r}")
        self.dropout_engine = engine
        self.encode_layer_dims = [self.item_num] + self.layers + [self.lat_dim]
        self.decode_layer_dims = [int(self.lat_dim / 2)] + self.encode_layer_dims[::-1][1:]

        hist_id = torch.as_tensor(config['history_item_id'])
        hist_val = torch.as_tensor(config['history_item_value'])
        if hist_id.shape[0] != self.user_num or hist_val.shape != hist_id.shape:
            raise ValueError(f"history_item_id / history_item_value must both be [user_num={self.user_num}, max_len]")
        self._check_ids((hist_id,), (self.item_num,), ('history item',))
        self.history_item_id = hist_id.to(self.device, torch.int64).contiguous()
        self.history_item_value = hist_val.to(self.device, torch.float32).contiguous()
        self._input = ops.VaeInput(self.history_item_id, self.history_item_value, self.item_num)

        # reference RNG stream (:50-69): each nn.Linear draws its own reset at construction, in module order; then
        # apply(_init_weight) re-draws every weight in the same order and zeroes every bias (AbstractRecommender.py:69-77)
        import torch.nn as nn
        dims = [self.encode_layer_dims, self.decode_layer_dims]
        linears = [[nn.Linear(a, b) for a, b in zip(d[:-1], d[1:])] for d in dims]
        init = _INIT[self.initializer]
        with torch.no_grad():
            parts = []
            for side in linears:
                for lin in side:
                    init(lin.weight)
                    lin.bias.zero_()
            for k, lin in enumerate(linears[0] + linears[1]):
                w = lin.weight.t() if k == 0 else lin.weight
                parts += [w.contiguous().reshape(-1), lin.bias.reshape(-1)]
            net = torch.cat(parts)
        assert net.numel() == ops.vae_param_count(self.item_num, self.layers, self.lat_dim)
        self.net = net.to(self.device)
        self._views = self._param_views()
        self._score_ws = None

    # ------------------------------------------------------------------ state
    def _param_views(self):
        views, off = {}, 0
        for side, dims in (('encoder', self.encode_layer_dims), ('decoder', self.decode_layer_dims)):
            for k, (a, b) in enumerate(zip(dims[:-1], dims[1:])):
                w = self.net[off:off + a * b]
                views[f'{side}.{2 * k}.weight'] = w.view(a, b).t() if side == 'encoder' and k == 0 else w.view(b, a)
                off += a * b
                views[f'{side}.{2 * k}.bias'] = self.net[off:off + b]
                off += b
        return views

    def state_dict(self):
        return dict(self._views)

    def parameters(self):
        return list(self._views.values())

    def load_state_dict(self, sd):
        for k, t in self._views.items():
            t.copy_(torch.as_tensor(sd[k]).reshape(t.shape))

    # ------------------------------------------------------------------ steps
    def _hyper(self, opt=None):
        return ops.hyper(self.lr, 0.0, 0.0, opt or self._optimizer_name())

    def _begin_fit(self, opt):
        self._hp = self._hyper(opt)
        self._opt_steps = 0
        self._fit_opt = opt
        self._ws = None

    def _ensure(self, rows=0):
        """Optimiser state and scratch for steps of up to ``rows`` users; a step outside fit() starts a fresh optimiser.  A
        larger batch than the workspace was built for grows it, keeping the optimiser state."""
        if self._hp is None:
            self._begin_fit(self._optimizer_name())
        if self._ws is None:
            self._ws = ops.VaeWorkspace(self.item_num, self.layers, self.lat_dim, self._fit_opt, rows, self._input.max_row_len,
                                        self.device)
        elif self._ws.max_rows < rows:
            self._ws = self._ws.grown(rows)

    def _host_draws(self, B, n_steps):
        """Per step, the draws of the reference's forward() on the global CPU generator: F.dropout's keep mask [B, I] (bit-packed,
        bit b * I + i), then randn_like(std) [B, lat // 2] -> (int32 CUDA words [n_steps * words], fp32 CUDA eps)."""
        words = ops.vae_keep_words(B, self.item_num)
        bits = np.zeros((n_steps, words), dtype=np.int32) if self.dropout > 0.0 else None
        eps = torch.empty(n_steps, B, self.lat_dim // 2, dtype=torch.float32)
        for s in range(n_steps):
            if bits is not None:
                keep = torch.empty(B, self.item_num, dtype=torch.float32).bernoulli_(1 - self.dropout)
                packed = np.packbits(keep.numpy().reshape(-1).astype(bool), bitorder='little')
                bits[s].view(np.uint8)[:packed.size] = packed
            eps[s] = torch.randn(B, self.lat_dim // 2)
        return (None if bits is None else torch.from_numpy(bits.reshape(-1)).to(self.device)), eps.to(self.device)

    def _launch(self, users, batch, first, n_steps, apply=True):
        """n_steps steps over the device users (int64) in batches of ``batch``; advances ``update`` by the steps run."""
        kw = dict(apply=apply, training=self.training, total_anneal_steps=self.total_anneal_steps,
                  anneal_cap=float(self.anneal_cap), dropout=self.dropout)
        run = lambda us, b, f, k, step0, **extra: ops.vae_train_steps(  # noqa: E731
            self.net, self._ws, self._input, us, b, f, k, self._hp, adam_step0=step0, update0=self.update, **kw, **extra)
        out = []
        if not self.training or self.dropout_engine == 'philox':
            seed = int(torch.randint(0, 2 ** 62, ()).item()) if self.training else 0
            losses = run(users, batch, first, n_steps, self._opt_steps, seed=seed)
            self.update += n_steps
            return losses
        per_step = batch * self.item_num // 8 + batch * self.lat_dim * 2 + 1
        chunk = max(1, (64 << 20) // per_step)                          # at most 64 MB of host draws per call
        s = first
        while s < first + n_steps:
            k = min(chunk, first + n_steps - s)
            full, last = ragged_split(users.numel(), batch, s, k)
            step0 = self._opt_steps + (s - first)
            if full > 0:
                bits, eps = self._host_draws(batch, full)
                out.append(run(users, batch, s, full, step0, keep_bits=bits, eps=eps))
                self.update += full
            if last:
                base = (s + full) * batch
                bits, eps = self._host_draws(last, 1)
                out.append(run(users[base:], last, 0, 1, step0 + full, keep_bits=bits, eps=eps))
                self.update += 1
            s += k
        return torch.cat(out)

    def _train_steps(self, users, batch, first, n_steps):
        self._ensure(batch)
        losses = self._launch(users, batch, first, n_steps, apply=True)
        self._opt_steps += n_steps
        return losses

    def _batch_users(self, batch):
        users = torch.as_tensor(batch).reshape(-1)
        return self._device_ids((users,), (self.user_num,), ('user',), torch.int64)[0]

    def calc_loss(self, batch):
        """0-d fp32 loss of one batch of users (:92-110), in the current mode; advances ``update``; no parameter changes."""
        users = self._batch_users(batch)
        self._ensure(users.numel())
        return self._launch(users, users.numel(), 0, 1, apply=False).to(torch.float32).reshape(())

    def train_step(self, batch):
        """zero_grad + calc_loss + backward + optimizer.step on one batch of users, in train mode -> loss.item()."""
        users = self._batch_users(batch)
        was = self.training
        self.train()
        try:
            return float(self._train_steps(users, users.numel(), 0, 1).item())
        finally:
            self.train(was)

    def _loader_plan(self, train_loader):
        return loader_plan(train_loader, _int_rows)

    def _fit_epoch_bulk(self, plan, epoch):
        data, bs, shuffle, drop_last, gen = plan
        T = data.shape[0]
        key = (id(data), fingerprint(data))
        if getattr(self, '_users_key', None) != key:
            self._check_ids((data,), (self.user_num,), ('user',))
            self._users_dev = torch.from_numpy(np.ascontiguousarray(data, dtype=np.int64)).to(self.device)
            self._users_key = key
        d_perm = self._device_permutation(T, shuffle, gen)
        users = self._users_dev if d_perm is None else self._users_dev[d_perm]
        n_use = (T // bs) * bs if drop_last else T
        nsteps = (n_use + bs - 1) // bs
        if nsteps == 0:
            return 0.
        losses = self._train_steps(users[:n_use].contiguous(), bs, 0, nsteps)     # raises ValueError on NaN
        return float(losses.sum().item())

    # ------------------------------------------------------------------ scoring (eval mode)
    def _scores(self, users, cands=None):
        if self._score_ws is None:
            rows = min(self.SCORE_ROWS, self.user_num)
            self._score_ws = ops.VaeWorkspace(self.item_num, self.layers, self.lat_dim, None, rows, self._input.max_row_len,
                                              self.device)
        return ops.vae_scores(self.net, self._score_ws, self._input, users, cands)

    def predict(self, u, i):
        """-> python float: the eval-mode logit of item i for user u (:112-119)."""
        us, its = self._device_ids(([u], [i]), (self.user_num, self.item_num), ('user', 'item'), torch.int64)
        return float(self._scores(us, its.reshape(1, 1)).item())

    def rank(self, test_loader):
        """-> float32 ndarray [n_test_users, topk] of the top candidates by eval-mode logit (:121-138)."""
        ins = self._rank_inputs(test_loader)
        if ins is None:
            return np.zeros((0,), np.float32)
        users, cands, k = ins
        d_cands = torch.from_numpy(cands).to(self.device)
        scores = self._scores(torch.from_numpy(users).to(self.device), d_cands)
        return ops.topk_from_scores(scores, d_cands, k).cpu().numpy()

    def full_rank(self, u):
        """-> int64 ndarray [topk] of the top items of user u over the full logit row; no masking of train items (:140-145)."""
        users = self._device_ids(([int(u)],), (self.user_num,), ('user',), torch.int64)[0]
        return ops.topk_from_scores(self._scores(users), None, min(self.topk, self.item_num))[0].cpu().numpy()
