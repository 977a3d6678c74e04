"""Restatement of the Multi-VAE device path (csrc/vae.cu) in numpy / torch float64, for the tests.  It does not import the
reference.

- ``input_rows``: the rows get_user_rating_matrix builds (index_put_ without accumulate: the last slot naming an item wins).
- ``host_draws``: what the reference's forward() draws per train step on the global CPU generator (F.dropout's keep mask,
  then randn_like(std)); the device path's parity mode consumes exactly these.
- ``Vae``: the network on a flat-free dict of float64 tensors with the reference's keys; ``step`` is calc_loss + backward +
  optimizer.step (torch.optim.Adam / SGD on the float64 tensors), ``scores`` the eval-mode logits.
- ``fit``: the driver loop with the DataLoader's RNG protocol (``epoch_order``, restated from torch.utils.data).
"""
import math

import numpy as np
import torch


def input_rows(hist_id, hist_val, item_num):
    """dense float64 [U, I]: (u, i) = value of the last slot of row u naming i (0 where none or where that value is 0)."""
    hid, hval = np.asarray(hist_id), np.asarray(hist_val, np.float64)
    U, L = hid.shape
    flat = (np.arange(U)[:, None] * item_num + hid).reshape(-1)
    rev = flat[::-1]
    _, first_rev = np.unique(rev, return_index=True)
    last = len(flat) - 1 - first_rev
    X = np.zeros(U * item_num)
    X[flat[last]] = hval.reshape(-1)[last]
    return X.reshape(U, item_num)


def host_draws(B, item_num, half, dropout):
    """-> (keep float [B, I] or None, eps [B, half]) drawn as the reference's forward() draws them."""
    keep = torch.empty(B, item_num, dtype=torch.float32).bernoulli_(1 - dropout) if dropout > 0 else None
    eps = torch.randn(B, half)
    return keep, eps


class Vae:
    def __init__(self, state, hidden, latent_dim, item_num, opt, lr, dropout, anneal_cap, total_anneal_steps):
        self.p = {k: torch.tensor(np.asarray(v), dtype=torch.float64, requires_grad=True) for k, v in state.items()}
        self.ne = self.nd = len(hidden) + 1
        self.lat, self.half, self.I = latent_dim, latent_dim // 2, item_num
        self.dropout, self.cap, self.total = dropout, anneal_cap, total_anneal_steps
        params = list(self.p.values())
        self.opt = torch.optim.Adam(params, lr=lr) if opt == 'adam' else torch.optim.SGD(params, lr=lr)
        self.update = 0

    def _mlp(self, side, n, h):
        for k in range(n):
            h = h @ self.p[f'{side}.{2 * k}.weight'].T + self.p[f'{side}.{2 * k}.bias']
            if k < n - 1:
                h = torch.tanh(h)
        return h

    def forward(self, R, keep=None, eps=None):
        h = R / R.norm(dim=1, keepdim=True).clamp_min(1e-12)
        if keep is not None:
            h = h * keep.to(torch.float64) / (1 - self.dropout)
        h = self._mlp('encoder', self.ne, h)
        mu, logvar = h[:, :self.half], h[:, math.ceil(self.lat / 2):]
        z = mu if eps is None else eps.to(torch.float64) * torch.exp(0.5 * logvar) + mu
        return self._mlp('decoder', self.nd, z), mu, logvar

    def loss(self, R, keep=None, eps=None):
        self.update += 1
        anneal = min(self.cap, 1. * self.update / self.total) if self.total > 0 else self.cap
        z, mu, logvar = self.forward(R, keep, eps)
        kl = -0.5 * torch.mean(torch.sum(1 + logvar - mu.pow(2) - logvar.exp(), dim=1)) * anneal
        ce = -(torch.log_softmax(z, 1) * R).sum(1).mean()
        return ce + kl

    def step(self, R, keep=None, eps=None):
        self.opt.zero_grad()
        loss = self.loss(R, keep, eps)
        loss.backward()
        self.opt.step()
        return float(loss.item())

    def scores(self, R):
        with torch.no_grad():
            return self.forward(R)[0].numpy()

    def state(self):
        return {k: v.detach().numpy().copy() for k, v in self.p.items()}


def epoch_order(n):
    """The index order of one epoch of ``DataLoader(ds, shuffle=True)`` with its global-RNG draws: the iterator's base seed
    (torch/utils/data/dataloader.py), then RandomSampler's generator seed and torch.randperm on that generator
    (torch/utils/data/sampler.py)."""
    torch.empty((), dtype=torch.int64).random_()
    seed = int(torch.empty((), dtype=torch.int64).random_().item())
    g = torch.Generator()
    g.manual_seed(seed)
    return torch.randperm(n, generator=g).numpy()


def fit(model, X, data, batch_size, epochs, draws=host_draws):
    """The reference's fit over ``DataLoader(AEDataset, batch_size, shuffle=True)``: -> per-step losses."""
    X = torch.from_numpy(np.asarray(X, np.float64))
    data = np.asarray(data)
    losses = []
    for _ in range(epochs):
        perm = epoch_order(len(data))
        for s in range(0, len(data), batch_size):
            users = torch.from_numpy(data[perm[s:s + batch_size]].astype(np.int64))
            keep, eps = draws(len(users), model.I, model.half, model.dropout)
            losses.append(model.step(X[users], keep, eps))
    return np.array(losses)


def init_state(item_num, hidden, latent_dim):
    """The reference's init stream (nn.Linear resets in module order, then xavier_normal_ on every weight, zero biases) on the
    global CPU generator -> state dict of float32 arrays with the reference's keys."""
    enc = [item_num] + list(hidden) + [latent_dim]
    dec = [latent_dim // 2] + enc[::-1][1:]
    sides = [('encoder', [torch.nn.Linear(a, b) for a, b in zip(enc[:-1], enc[1:])]),
             ('decoder', [torch.nn.Linear(a, b) for a, b in zip(dec[:-1], dec[1:])])]
    out = {}
    with torch.no_grad():
        for side, lins in sides:
            for k, lin in enumerate(lins):
                torch.nn.init.xavier_normal_(lin.weight, gain=1.0)
                out[f'{side}.{2 * k}.weight'] = lin.weight.numpy().copy()
                out[f'{side}.{2 * k}.bias'] = np.zeros(lin.out_features, np.float32)
    return out
