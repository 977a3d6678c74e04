"""Multi-VAE: teacher-forced steps of drb_vae_train_steps and the eval-mode scores of drb_vae_scores against a float64 reference,
on the shared harness (fp64_step.py).

The reference runs the step of csrc/vae.cu (the oracle's network, oracle/vae_oracle.py) on a snapshot of the device's flat
parameter block and optimiser state, with the same host-drawn keep mask and normals, and carries each value's noise scale N
along the chain: a product adds the sum of |contributions|; tanh, exp, log and the softmax carry N through their derivative
and add their own rounding; the row L2 norm, the log-sum-exp over I logits and the bias column sums add one rounding per
term.  There is no discrete part (fp32 throughout, and tanh has no kink): P = 0.  It reads only the batch's input rows, and
runs the output layer (the [B, I] logits, the softmax cross-entropy and the layer's gradients) in blocks of ROW_BLOCK rows,
so that a B = 4 096 step at I = 26 744 never holds the dozen [B, I] float64 arrays of that layer at once.

Cases: the two fixture networks of tests/golden/vae.npz; a geometry sweep over the kernels' edges (the output layer's k
slices at I = 1 024, 1 025, 4 099, 16 384 and 16 385, hidden widths 3, 65, 257, [600, 200] and eight layers, latent sizes 2 and
129, batches of 1, 64, 65, 257 and 32 768 rows, input rows longer than 256 nonzeros, empty, real-valued, or with item 0 erased
by the padding, a user twice in one batch); and the ML-20M bench shape (utils.synthetic.make_interactions(138493, 26744,
20_000_000), hidden [600], latent 128, dropout 0.5) at B = 256 and 4 096: three steps each under SGD and Adam, one 3-step
launch against three single launches, one step run twice from one snapshot (bitwise equal), and the eval-mode logits of 256
users over every item and of 4 096 users over 1 000 candidates, per element |s - s64| <= KAPPA u N, ranked through
VAECF.rank / full_rank.

Calibrated on one H100 80GB HBM3 (700 W power limit).  "Needed" is the per-element KAPPA of an SGD step; every Adam step of
every case passes at the ladder's lowest rung 0.125.  At KAPPA = 0.25:
- fixture cases: needed 0.029 (case a; 0.0015 in case b); worst error / bound 0.40 (Adam), 0.39 (SGD);
- geometry sweep: needed 0.072 (I = 16 384, hidden [257]; <= 0.035 elsewhere); worst error / bound 0.46 (SGD, B = 32 768),
  0.42 (Adam, eight layers);
- bench shape steps: needed 0.022 (B = 4 096; 0.0054 at B = 256); worst error / bound 0.10 (SGD), 0.50 (Adam, B = 4 096);
  the 3-step launch ends bitwise equal to the three single launches, and the repeated B = 4 096 Adam step is bitwise equal;
- bench shape scores: worst error / bound 0.021 (every item of 256 users), 0.0084 (4 096 users x 1 000 candidates); rank
  and full_rank equal the stable sort of the device's scores and agree with the float64 order.
There the new (sweep and bench shape) cases take 37 s of wall time, the bench-shape draw included.  The CPU part runs the
same checks with the reference in float32 standing in for the device (rehearsal) on the fixture and the small sweep cases,
and shows that a 1e-3 relative error in the output layer's gradient, a dropped last k slice of the output layer's input
gradient, and a batch row missing from the layer-0 weight gradient each fail them.
"""
import functools
import math
import os
import sys
import time
from types import SimpleNamespace

import numpy as np
import pandas as pd
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fp64_step  # noqa: E402
from fp64_step import F64, Stepper, U_RND, checked_step, launch_vs_singles, report, summary  # noqa: E402
from oracle import vae_oracle as vo  # noqa: E402
from conftest import golden  # noqa: E402

KAPPA = 0.25
ROW_BLOCK = 1024          # rows of the output layer's [B, I] arrays the reference holds at once


def _layers(I, hidden, lat):
    """[(side, k, in, out, w_off, b_off)] of the flat block, the first encoder weight item-major"""
    enc = [I] + list(hidden) + [lat]
    dec = [lat // 2] + enc[::-1][1:]
    out, off = [], 0
    for side, dims in (("encoder", enc), ("decoder", dec)):
        for k, (a, b) in enumerate(zip(dims[:-1], dims[1:])):
            out.append((side, k, a, b, off, off + a * b))
            off += a * b + b
    return out, off


def last_slice_start(I):
    """the first column of the last of vae.cu's k slices of the output layer's input gradient (gemm_nn_slices)"""
    S = min(16, (I + 1023) // 1024)
    chunk = ((I + S - 1) // S + 15) // 16 * 16
    return ((I + chunk - 1) // chunk - 1) * chunk


def dense_rows(hist_id, hist_val, users, I, dt=F64):
    """the input rows of `users` as the device's input CSR holds them (index_put_ without accumulate: the last slot naming an
    item wins, so the (0, 0.0) padding erases item 0 of a short row) -> dense [B, I] on the history's device"""
    ids, vals = hist_id[users], hist_val[users].to(dt)
    B, L = ids.shape
    flat = (torch.arange(B, device=ids.device)[:, None] * I + ids).reshape(-1)
    slot = torch.arange(B * L, device=ids.device)
    last = torch.full((B * I,), -1, dtype=torch.int64, device=ids.device).scatter_reduce_(0, flat, slot, "amax")
    win = last[flat] == slot
    R = torch.zeros(B * I, dtype=dt, device=ids.device)
    R[flat[win]] = vals.reshape(-1)[win]
    return R.view(B, I)


def _wb(W, lay, L):
    side, k, a, b, wo, bo = lay[L]
    w = W[wo:wo + a * b].view(a, b).T if L == 0 else W[wo:wo + a * b].view(b, a)
    return w, W[bo:bo + b]


def _linear(W, lay, L, h, hN):
    w, b = _wb(W, lay, L)
    z = h @ w.T + b
    return z, (h.abs() + hN) @ w.abs().T + b.abs() + z.abs()


def _tanh(h, hN):
    a = torch.tanh(h)
    return a, (1 - a * a) * hN + a.abs()


def vae_forward(net, R, I, hidden, lat, dropout=0.0, keep=None, eps=None, dt=F64, logits=True):
    """the forward pass with its noise on the batch's input rows R -> namespace: encoder activations `acts` (the dropped input
    first), mu / logvar, the normals e and std, decoder activations `dacts` (z first, up to the output layer's input) and, with
    logits, `logit` / `logitN`.  Eval mode (what drb_vae_scores computes): keep = eps = None, z = mu."""
    lay, _ = _layers(I, hidden, lat)
    W = net.to(dt)
    R = R.to(dt)
    A = lambda x: x.abs()  # noqa: E731
    half, lo = lat // 2, lat - lat // 2
    nnz = (R != 0).sum(1, keepdim=True).to(dt)
    x = R / R.norm(dim=1, keepdim=True).clamp_min(1e-12)
    if keep is not None:
        x = x * keep.to(dt) * float(np.float32(1.0 / (1.0 - dropout)))
    xN = A(x) * (nnz + 2)
    ne = nd = len(hidden) + 1
    acts = [(x, xN)]
    h, hN = x, xN
    for L in range(ne):
        h, hN = _linear(W, lay, L, h, hN)
        if L < ne - 1:
            h, hN = _tanh(h, hN)
        acts.append((h, hN))
    mu, muN = h[:, :half], hN[:, :half]
    lv, lvN = h[:, lo:], hN[:, lo:]
    std = torch.exp(0.5 * lv)
    if eps is None:
        e, z, zN = torch.zeros_like(mu), mu, muN
    else:
        e = eps.to(R.device).to(dt)
        z = e * std + mu
        zN = A(e) * std * (0.5 * lvN + 1) + muN + A(z)
    dacts = [(z, zN)]
    for l in range(nd - 1):
        h, hN = _tanh(*_linear(W, lay, ne + l, *dacts[-1]))
        dacts.append((h, hN))
    f = SimpleNamespace(W=W, lay=lay, R=R, nnz=nnz, acts=acts, mu=mu, muN=muN, lv=lv, lvN=lvN, e=e, std=std, dacts=dacts)
    if logits:
        f.logit, f.logitN = _linear(W, lay, ne + nd - 1, *dacts[-1])
    return f


def vae_ref(net, R, I, hidden, lat, dropout, anneal, dt=F64, defects=(), keep=None, eps=None):
    """one train step's gradient, its noise N, the loss and its noise on the batch's input rows R -> harness result (P = 0).
    defects (rehearsal only): "grad_scale" the output layer's dz 1e-3 too large; "drop_last_slice" the last k slice's share of
    the output layer's input gradient dropped; "drop_last_row_dw0" the last batch row missing from the layer-0 weight gradient"""
    f = vae_forward(net, R, I, hidden, lat, dropout, keep, eps, dt, logits=False)
    W, lay, R, nnz = f.W, f.lay, f.R, f.nnz
    dev = W.device
    A = lambda x: x.abs()  # noqa: E731
    _, nW = _layers(I, hidden, lat)
    half, lo = lat // 2, lat - lat // 2
    B = R.shape[0]
    ne = nd = len(hidden) + 1
    mu, muN, lv, lvN, e, std = f.mu, f.muN, f.lv, f.lvN, f.e, f.std
    g = torch.zeros(nW, dtype=dt, device=dev)
    N = torch.zeros(nW, dtype=F64, device=dev)

    def put(L, gw, gwN, gb, gbN):
        side, k, a, b, wo, bo = lay[L]
        if L == 0:
            gw, gwN = gw.T, gwN.T
        g[wo:wo + a * b] = gw.reshape(-1)
        N[wo:wo + a * b] = gwN.reshape(-1).to(F64)
        g[bo:bo + b] = gb
        N[bo:bo + b] = gbN.to(F64)

    # output layer, in blocks of rows: logits, log-softmax cross-entropy, dz = (softmax sum(r) - r) / B in place of the logits,
    # then its weight / bias gradients (sums over rows, so the blocks add up) and its input gradient (per row)
    Lo = ne + nd - 1
    a, aN = f.dacts[-1]
    w, _ = _wb(W, lay, Lo)
    H = w.shape[1]
    cut = last_slice_start(I) if "drop_last_slice" in defects else I
    gw, gwN = torch.zeros(I, H, dtype=dt, device=dev), torch.zeros(I, H, dtype=dt, device=dev)
    gb, gbN = torch.zeros(I, dtype=dt, device=dev), torch.zeros(I, dtype=dt, device=dev)
    da, daN = torch.empty(B, H, dtype=dt, device=dev), torch.empty(B, H, dtype=dt, device=dev)
    ce_row, ce_rowN = torch.empty(B, dtype=dt, device=dev), torch.empty(B, dtype=dt, device=dev)
    for r0 in range(0, B, ROW_BLOCK):
        r = slice(r0, min(B, r0 + ROW_BLOCK))
        logit, logitN = _linear(W, lay, Lo, a[r], aN[r])
        Rb, nz = R[r], nnz[r]
        lse = torch.logsumexp(logit, 1, keepdim=True)
        p = torch.exp(logit - lse)
        lseN = (p * logitN).sum(1, keepdim=True) + I
        ls = logit - lse
        lsN = logitN + lseN + A(ls)
        del logit, logitN
        rs = Rb.sum(1, keepdim=True)
        ce_row[r] = (Rb * ls).sum(1)
        ce_rowN[r] = (A(Rb) * lsN).sum(1)
        dz = (p * rs - Rb) / B
        if "grad_scale" in defects:
            dz = dz * (1 + 1e-3)
        dzN = (p * (lsN + 1) * A(rs) + p * A(rs) * nz) / B + A(dz)
        del p, ls, lsN
        gw += dz.T @ a[r]
        gwN += (A(dz) + dzN).T @ A(a[r]) + A(dz).T @ aN[r]
        gb += dz.sum(0)
        gbN += (A(dz) + dzN).sum(0)
        full = dz @ w
        da[r] = full if cut == I else dz[:, :cut] @ w[:cut]
        daN[r] = (A(dz) + dzN) @ A(w) + A(full)
    put(Lo, gw, gwN, gb, gbN)
    del gw, gwN
    kl_t = 1 + lv - mu * mu - torch.exp(lv)
    kl_row = kl_t.sum(1)
    kl_rowN = (1 + A(lv) + lvN + mu * mu + 2 * A(mu) * muN + torch.exp(lv) * (1 + lvN)).sum(1)
    loss = -ce_row.mean() + (-0.5 * kl_row.mean()) * anneal
    lossN = float(ce_rowN.mean() + 0.5 * anneal * kl_rowN.mean() + A(loss) * 4)

    def tanh_back(da, daN, a, aN):
        return da * (1 - a * a), daN * (1 - a * a) + A(da) * 2 * A(a) * aN + A(da * (1 - a * a))

    cur, curN = (tanh_back(da, daN, a, aN) if nd > 1 else (da, daN))
    for l in range(nd - 2, -1, -1):
        L = ne + l
        w, _ = _wb(W, lay, L)
        a, aN = f.dacts[l]
        put(L, cur.T @ a, (A(cur) + curN).T @ A(a) + A(cur).T @ aN, cur.sum(0), (A(cur) + curN).sum(0))
        da = cur @ w
        daN = (A(cur) + curN) @ A(w) + A(da)
        cur, curN = tanh_back(da, daN, a, aN) if l > 0 else (da, daN)
    dzl, dzlN = cur, curN
    dmu = dzl + anneal * mu / B
    dmuN = dzlN + anneal * muN / B + A(dmu)
    dlv = dzl * e * std * 0.5 + anneal * 0.5 * (torch.exp(lv) - 1) / B
    dlvN = (dzlN + A(dzl) * 0.5 * lvN) * A(e) * std * 0.5 + anneal * torch.exp(lv) * (1 + lvN) / (2 * B) + A(dlv)
    cur = torch.zeros(B, lat, dtype=dt, device=dev)
    curN = torch.zeros(B, lat, dtype=dt, device=dev)
    cur[:, :half], cur[:, lo:] = dmu, dlv
    curN[:, :half], curN[:, lo:] = dmuN, dlvN
    for L in range(ne - 1, -1, -1):
        a, aN = f.acts[L]
        gw = cur[:-1].T @ a[:-1] if L == 0 and "drop_last_row_dw0" in defects else cur.T @ a
        put(L, gw, (A(cur) + curN).T @ A(a) + A(cur).T @ aN, cur.sum(0), (A(cur) + curN).sum(0))
        if L > 0:
            w, _ = _wb(W, lay, L)
            da = cur @ w
            cur, curN = tanh_back(da, (A(cur) + curN) @ A(w) + A(da), a, aN)
    zero = torch.zeros_like(N)
    return dict(g={"net": g.to(F64)}, N={"net": N}, P={"net": zero}, loss=float(loss), lossN=lossN, lossP=0.0, flagged=0.0)


class _Model:
    phi_max = 0.0
    ladder = True
    ref_uses_kappa = False

    def _model(self, I, hidden, lat, hist_id, hist_val, dropout, anneal):
        self.I, self.hidden, self.lat, self.dropout, self.anneal = I, list(hidden), lat, dropout, anneal
        self.hist = {"cpu": (torch.as_tensor(hist_id, dtype=torch.int64), torch.as_tensor(hist_val, dtype=torch.float32))}
        self.kappa = KAPPA

    def rows(self, users, dt=F64):
        """the users' dense input rows on the users' device"""
        key = str(users.device)
        if key not in self.hist:
            self.hist[key] = tuple(t.to(users.device) for t in self.hist["cpu"])
        return dense_rows(*self.hist[key], users, self.I, dt)

    def reference(self, pre, idx, kappa, dt=F64, defects=(), keep=None, eps=None):
        dev = pre["net"].device
        kp = None if keep is None else keep.to(dev)
        return vae_ref(pre["net"], self.rows(idx[0].to(dev), dt), self.I, self.hidden, self.lat, self.dropout, self.anneal, dt,
                       defects, kp, eps)

    def sections(self):
        lay, _ = _layers(self.I, self.hidden, self.lat)
        out = []
        for side, k, a, b, wo, bo in lay:
            out.append((f"{side}.{2 * k}.weight", "net", wo, wo + a * b, b if (side, k) == ("encoder", 0) else a))
            out.append((f"{side}.{2 * k}.bias", "net", bo, bo + b, 1))
        return out


class VaeGpu(_Model, Stepper):
    device = "cuda"

    def __init__(self, I, hidden, lat, net, hist_id, hist_val, users, opt, lr, dropout, anneal_cap, max_rows=None):
        from daisyrec_b200 import ops
        self.ops, self.opt, self.lr = ops, opt, lr
        self._model(I, hidden, lat, hist_id, hist_val, dropout, anneal_cap)
        self.net = torch.from_numpy(np.asarray(net, np.float32)).cuda().contiguous()
        self.t = dict(net=self.net)
        self.planes = (torch.from_numpy(np.asarray(users, np.int64)).cuda(),)
        hid, hval = self.hist["cpu"]
        self.inp = ops.VaeInput(hid.cuda(), hval.cuda(), I)
        self.hp = ops.hyper(lr, 0.0, 0.0, opt)
        rows = max_rows or min(self.planes[0].numel(), ops.VAE_MAX_ROWS)
        self.ws = ops.VaeWorkspace(I, hidden, lat, opt, rows, self.inp.max_row_len, "cuda")
        self.draws = None                       # (keep, eps) every step of a multi-step launch uses
        nW = self.net.numel()
        a = (4 * nW + 255) // 256 * 256
        if opt == "adam":
            f = self.ws.buf[256 + a:256 + 3 * a].view(torch.float32)
            self.mom = {"net": (f[:nW], f[a // 4:a // 4 + nW])}

    def run(self, lo, n, batch, k, adam_step0=0, apply=True, first_step=0, keep=None, eps=None):
        """k == 1: one step on rows [lo, lo + n); k > 1: steps first_step .. of `batch` rows over rows [lo, lo + n), each with
        the same draws (self.draws)"""
        if keep is None and eps is None:
            keep, eps = self.draws
        b = n if k == 1 else batch
        users = self.planes[0][lo:lo + n]
        bits = None
        if keep is not None:
            packed = np.packbits(keep.numpy().reshape(-1).astype(bool), bitorder="little")
            w = np.zeros(self.ops.vae_keep_words(b, self.I) * 4, np.uint8)
            w[:packed.size] = packed
            bits = torch.from_numpy(np.tile(w.view(np.int32), k)).cuda()
        e = eps.reshape(1, b, -1).expand(k, -1, -1).contiguous().cuda()
        out = self.ops.vae_train_steps(self.net, self.ws, self.inp, users, b, first_step, k, self.hp,
                                       adam_step0=adam_step0 + first_step, apply=apply, training=True, total_anneal_steps=0,
                                       anneal_cap=self.anneal, dropout=self.dropout, keep_bits=bits, eps=e)
        torch.cuda.synchronize()
        return out.cpu().numpy()


class StandIn(_Model, fp64_step.StandIn):
    def __init__(self, I, hidden, lat, net, hist_id, hist_val, users, opt, lr, dropout, anneal_cap, defects=()):
        super().__init__(dict(net=net), (users,), opt, lr, 0.0, defects)
        self._model(I, hidden, lat, hist_id, hist_val, dropout, anneal_cap)

    def stand_in_ref(self, idx, keep=None, eps=None):
        return self.reference(self.t, idx, self.kappa, torch.float32, self.defects, keep, eps)


# ---------------------------------------------------------------- problems
def _init_net(rng, I, hidden, lat):
    """xavier-normal weights and small nonzero biases in the flat block"""
    lay, nW = _layers(I, hidden, lat)
    net = np.empty(nW, np.float32)
    for side, k, a, b, wo, bo in lay:
        net[wo:wo + a * b] = rng.standard_normal(a * b, np.float32) * np.float32(math.sqrt(2.0 / (a + b)))
        net[bo:bo + b] = rng.standard_normal(b, np.float32) * np.float32(0.1)
    return net


def _history(rows, vals):
    """(item ids, values) per user -> the padded history matrices of get_history_matrix (padding (0, 0.0))"""
    L = max(1, max(len(r) for r in rows))
    hid, hval = np.zeros((len(rows), L), np.int64), np.zeros((len(rows), L), np.float32)
    for u, (r, v) in enumerate(zip(rows, vals)):
        hid[u, :len(r)], hval[u, :len(r)] = r, v
    return hid, hval


def _fixture(case):
    """the fixture's synthetic case: initial flat block, history, users in the fixture's first-appearance order"""
    g = golden("vae")
    p = f"s{case}_"
    U, I, lat = (int(x) for x in g[p + "meta"][:3])
    hidden = [int(h) for h in g[p + "hidden"]]
    keys = list(g[p + "keys"])
    lay, nW = _layers(I, hidden, lat)
    net = np.zeros(nW, np.float32)
    sd = {k: g[p + f"init{j}"] for j, k in enumerate(keys)}
    for side, k, a, b, wo, bo in lay:
        w = sd[f"{side}.{2 * k}.weight"]
        net[wo:wo + a * b] = (w.T if (side, k) == ("encoder", 0) else w).reshape(-1)
        net[bo:bo + b] = sd[f"{side}.{2 * k}.bias"]
    users = pd.Series(g[p + "df"][0]).unique().astype(np.int64)
    return SimpleNamespace(I=I, hidden=hidden, lat=lat, net=net, hist_id=g[p + "hist_id"], hist_val=g[p + "hist_val"],
                           users=users, batch=16, steps=(len(users) + 15) // 16)


# name: (I, hidden, latent, B, steps).  Each user set opens with a row of 300 nonzeros, an empty row, a row whose item 0 the
# padding erases and a row of half-star ratings; rows are half-star or binary; with B > 1 the batch's last user repeats its
# first.  I: 1 024 / 1 025 / 4 099 / 16 384 / 16 385 are 1, 2 (ragged), 5, 16 and 16 (capped) k slices of the output layer's
# input gradient; 257-wide layers take a second column pass in vae_enc0_kernel / vae_dw0_kernel / vae_colsum_kernel; B = 32 768
# is the largest batch (vae_dw0_kernel's shared-memory bitmap above the 48 KB default)
SWEEP = {
    "i1024": (1024, [3], 2, 64, 2),
    "i1025": (1025, [65], 129, 65, 2),
    "i4099": (4099, [40, 33, 65, 17, 24, 9, 48, 20], 16, 1, 3),
    "i16384": (16384, [257], 8, 257, 2),
    "i16385": (16385, [600, 200], 129, 64, 2),
    "b32768": (2048, [257], 10, 32768, 1),
}
SMALL = ("i1024", "i1025", "i4099")        # the sweep cases the CPU rehearsal runs


def _sweep(name):
    I, hidden, lat, B, steps = SWEEP[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    U = max(4, B * steps)
    rows, vals = [], []
    for u in range(U):
        n = (300, 0, 12, 40)[u] if u < 4 else int(rng.integers(1, 17))
        r = rng.choice(np.arange(1, I), n, replace=False)
        if u == 2:
            r[0] = 0                                            # item 0 in a short row: the padding erases it
        half = u == 3 or (u > 3 and rng.random() < 0.5)
        rows.append(r)
        vals.append(rng.integers(1, 11, n) / 2.0 if half else np.ones(n))
    hid, hval = _history(rows, vals)
    users = np.arange(U, dtype=np.int64)
    users[4:] = 4 + rng.permutation(U - 4)
    if B > 1:
        users[B - 1] = users[0]
    return SimpleNamespace(I=I, hidden=hidden, lat=lat, net=_init_net(rng, I, hidden, lat), hist_id=hid, hist_val=hval,
                           users=users[:B * steps], batch=B, steps=steps)


def _problem(case):
    return _fixture(case) if case in ("a", "b") else _sweep(case)


def _steps(st, pr, dropout, seed=0):
    torch.manual_seed(seed)
    recs = []
    n_rows = len(pr.users)
    for s in range(pr.steps):
        lo = s * pr.batch
        nb = min(pr.batch, n_rows - lo)
        keep, eps = vo.host_draws(nb, pr.I, pr.lat // 2, dropout)
        recs.append(checked_step(st, lo, nb, pr.batch, f"step {s}", adam_step0=s, ref_device=st.device, keep=keep, eps=eps))
    return recs


def _gpu(pr, users, opt, dropout, lr=None, max_rows=None):
    lr = lr or (0.05 if opt == "sgd" else 0.01)
    return VaeGpu(pr.I, pr.hidden, pr.lat, pr.net, pr.hist_id, pr.hist_val, users, opt, lr, dropout, 0.2, max_rows)


# case, optimiser, dropout: (a) one hidden layer, 34 warm users in steps of 16 (the third step is ragged), the user whose item 0
# the padding erases included; (b) two hidden layers, odd latent size 9; then the geometry sweep
CASES = ([("a", "sgd", 0.5), ("a", "adam", 0.5), ("b", "sgd", 0.0), ("b", "adam", 0.5)]
         + [(c, opt, 0.0 if c == "i16384" else 0.5) for c in SWEEP for opt in ("sgd", "adam")])
CPU_CASES = [c for c in CASES if c[0] in ("a", "b") + SMALL]


@pytest.mark.gpu
@pytest.mark.parametrize("case,opt,dropout", CASES)
def test_teacher_forced_step(case, opt, dropout):
    t0 = time.perf_counter()
    pr = _problem(case)
    st = _gpu(pr, pr.users, opt, dropout, max_rows=min(len(pr.users), 32768))
    recs = _steps(st, pr, dropout)
    report(f"vae {case} {opt} p={dropout}", recs)
    print(f"[vae {case} {opt}] {time.perf_counter() - t0:.1f} s")
    assert all(r["ok"] for r in recs)


@pytest.mark.parametrize("case,opt,dropout", CPU_CASES)
def test_rehearsal_on_stand_in(case, opt, dropout):
    """the GPU test body on the float32 reference standing in for the device"""
    pr = _problem(case)
    st = StandIn(pr.I, pr.hidden, pr.lat, pr.net, pr.hist_id, pr.hist_val, pr.users, opt, 0.05 if opt == "sgd" else 0.01,
                 dropout, 0.2)
    recs = _steps(st, pr, dropout)
    for r in recs:
        print(summary(r))
    assert all(r["ok"] for r in recs)


def test_rehearsal_flags_defective_stand_in():
    pr = _fixture("a")
    st = StandIn(pr.I, pr.hidden, pr.lat, pr.net, pr.hist_id, pr.hist_val, pr.users, "sgd", 0.05, 0.5, 0.2,
                 defects=("grad_scale",))
    pr.steps = 1
    recs = _steps(st, pr, 0.5)
    print(summary(recs[0]))
    assert not recs[0]["ok"]


@pytest.mark.parametrize("defect", ["drop_last_slice", "drop_last_row_dw0"])
def test_rehearsal_flags_defects_past_one_slice(defect):
    """at I = 1 025 (two k slices, the last one ragged): a dropped last k slice of the output layer's input gradient and a
    batch row missing from the layer-0 weight gradient each fail the step"""
    pr = _sweep("i1025")
    assert last_slice_start(pr.I) == 528
    st = StandIn(pr.I, pr.hidden, pr.lat, pr.net, pr.hist_id, pr.hist_val, pr.users, "sgd", 0.05, 0.5, 0.2, defects=(defect,))
    pr.steps = 1
    recs = _steps(st, pr, 0.5)
    print(summary(recs[0]))
    assert not recs[0]["ok"]


def test_dense_rows_keep_the_last_write():
    """the reference's input rows: the last slot naming an item wins, zero values (the padding) drop it"""
    hid = torch.tensor([[3, 0, 3, 1], [0, 2, 0, 0]])
    hval = torch.tensor([[1.0, 2.5, 4.0, 0.5], [1.5, 3.0, 0.0, 0.0]])
    R = dense_rows(hid, hval, torch.tensor([1, 0, 1]), 4)
    assert torch.equal(R, torch.tensor([[0, 0, 3.0, 0], [2.5, 0.5, 0, 4.0], [0, 0, 3.0, 0]], dtype=F64))
    assert torch.equal(dense_rows(hid, hval, torch.arange(2), 4), torch.from_numpy(vo.input_rows(hid.numpy(), hval.numpy(), 4)))


# ---------------------------------------------------------------- the ML-20M bench shape
BENCH_B, BENCH_STEPS = (256, 4096), 3


@functools.lru_cache(maxsize=1)
def _bench():
    """scripts/bench_vae.py's draw; the input restricted to the users the tests step on, renumbered: the first 3 x 4 096 users
    in first-appearance order with the draw's longest row at position 1 and position 3's user again at position 200"""
    from daisyrec_b200.utils.synthetic import make_interactions
    I, hidden, lat = 26744, [600], 128
    d = make_interactions(138493, I, 20_000_000)
    rp, col = d["row_ptr"].numpy(), d["col"].numpy()
    order = pd.Series(d["coo_u"].numpy()).unique().astype(np.int64)
    n = BENCH_STEPS * max(BENCH_B)
    longest = int(np.argmax(np.diff(rp)))
    sel = np.concatenate([order[:1], [longest], order[1:][order[1:] != longest][:n - 2]])
    sel[200] = sel[3]
    uniq, users = np.unique(sel, return_inverse=True)
    rows = [col[rp[u]:rp[u + 1]] for u in uniq]
    hid, hval = _history(rows, [np.ones(len(r)) for r in rows])
    assert hid.shape[1] == rp[longest + 1] - rp[longest] > 256
    rng = np.random.default_rng(2022)
    return SimpleNamespace(I=I, hidden=hidden, lat=lat, net=_init_net(rng, I, hidden, lat), hist_id=hid, hist_val=hval,
                           users=users.astype(np.int64), batch=None, steps=BENCH_STEPS)


@pytest.mark.gpu
@pytest.mark.parametrize("B", BENCH_B)
@pytest.mark.parametrize("opt", ["sgd", "adam"])
def test_bench_shape_steps(B, opt):
    """three consecutive teacher-forced steps at the bench shape: 16 k slices of 1 680 columns (the last 1 544), ragged
    64 x 64 GEMM tiles in every dimension (I = 26 744 = 56 mod 64, 600 = 24 mod 64), 26 744 logits per vae_ce_kernel row and
    a row of more than 256 nonzeros"""
    t0 = time.perf_counter()
    pr = _bench()
    pr = SimpleNamespace(**{**vars(pr), "batch": B, "users": pr.users[:B * BENCH_STEPS]})
    st = _gpu(pr, pr.users, opt, 0.5, lr=0.05 if opt == "sgd" else 1e-3, max_rows=B)
    recs = _steps(st, pr, 0.5)
    report(f"vae bench B={B} {opt}", recs)
    print(f"[vae bench B={B} {opt}] {time.perf_counter() - t0:.1f} s")


@pytest.mark.gpu
def test_bench_shape_launch_and_repeat():
    """one 3-step launch against three single launches at B = 256; one B = 4 096 Adam step run twice from one snapshot is
    bitwise equal (loss, parameters, moments)"""
    t0 = time.perf_counter()
    pr = _bench()
    B = 256
    torch.manual_seed(1)
    keep, eps = vo.host_draws(B, pr.I, pr.lat // 2, 0.5)
    multi, single = (_gpu(pr, pr.users[:3 * B], "sgd", 0.5, max_rows=B) for _ in range(2))
    multi.draws = (keep, eps)
    recs = launch_vs_singles(multi, single, 3 * B, B, 3, keep=keep, eps=eps)
    del multi, single
    B = 4096
    keep, eps = vo.host_draws(B, pr.I, pr.lat // 2, 0.5)
    runs = []
    for _ in range(2):
        st = _gpu(pr, pr.users[:B], "adam", 0.5, lr=1e-3, max_rows=B)
        loss = st.run(0, B, B, 1, keep=keep, eps=eps)
        runs.append((loss, st.net.clone(), *(m.clone() for m in st.mom["net"])))
        del st
    same = [np.array_equal(runs[0][0], runs[1][0])] + [torch.equal(a, b) for a, b in zip(runs[0][1:], runs[1][1:])]
    recs.append(dict(tag="B=4096 adam step twice", nb=B, loss=float(runs[0][0][0]), loss_ref=float("nan"), loss_ratio=0.0,
                     checks=dict(loss=same[0], net=same[1], m=same[2], v=same[3]), ok=all(same)))
    report("vae bench launches", recs)
    print(f"[vae bench launches] {time.perf_counter() - t0:.1f} s")


def _scores_ref(pr, net, users, rows_dev):
    """eval-mode float64 logits and their noise of `users`, [n, I] each"""
    out = [vae_forward(net, rows_dev(users[r0:r0 + ROW_BLOCK]), pr.I, pr.hidden, pr.lat)
           for r0 in range(0, len(users), ROW_BLOCK)]
    return torch.cat([f.logit for f in out]), torch.cat([f.logitN for f in out])


def _order_checks(ids_pos, s32, s64, bound):
    """top-K positions [n, K] against the device's fp32 scores (exact: a stable sort by score descending, then position) and
    the float64 scores (consecutive ids in the fp64 order unless their scores are within their bounds, and no id left out whose
    fp64 score lies above the last id's beyond both bounds) -> (exact, fp64)"""
    K = ids_pos.shape[1]
    want = torch.from_numpy(np.argsort(-s32.cpu().numpy(), axis=1, kind="stable")[:, :K].copy()).to(ids_pos.device)
    exact = bool(torch.equal(ids_pos, want))
    hi, lo = s64 + bound, s64 - bound
    got_hi, got_lo = hi.gather(1, ids_pos), lo.gather(1, ids_pos)
    ordered = bool((got_hi[:, :-1] >= got_lo[:, 1:]).all())
    left = torch.ones_like(s64, dtype=torch.bool).scatter_(1, ids_pos, False)
    missed = bool(((lo > got_hi[:, -1:]) & left).any())
    return exact, ordered and not missed


@pytest.mark.gpu
def test_bench_shape_scores_and_rank():
    """drb_vae_scores in eval mode at the bench shape against the float64 forward, per element |s - s64| <= KAPPA u N: every
    logit of 256 users (gemm_nt + bias) and 4 096 users x 1 000 candidates (vae_score_kernel), four passes of 1 024 rows; then
    VAECF.rank and full_rank on those scores: the ids equal a stable sort of the device's scores and agree with the float64
    order wherever the float64 scores are further apart than their bounds"""
    import logging
    from daisyrec_b200.model.VAECFRecommender import VAECF
    t0 = time.perf_counter()
    pr = _bench()
    users = torch.from_numpy(pr.users[:4096]).cuda()
    hist = tuple(torch.from_numpy(a).cuda() for a in (pr.hist_id, pr.hist_val))
    rows_dev = lambda u: dense_rows(*hist, u, pr.I)  # noqa: E731
    cfg = dict(mlp_hidden_size=pr.hidden, latent_dim=pr.lat, dropout=0.5, lr=0.001, total_anneal_steps=0, anneal_cap=0.2,
               epochs=1, optimizer='default', init_method='default', early_stop=False, topk=50, gpu='0',
               logger=logging.getLogger('vae-fp64'), UID_NAME='user', IID_NAME='item', user_num=len(pr.hist_id),
               item_num=pr.I, history_item_id=pr.hist_id, history_item_value=pr.hist_val)
    model = VAECF(cfg)
    model.net.copy_(torch.from_numpy(pr.net))
    model.eval()
    net = model.net
    rng = np.random.default_rng(7)
    cands = torch.from_numpy(rng.integers(0, pr.I, (4096, 1000))).cuda()
    full = model._scores(users[:256])
    cand = model._scores(users, cands)
    assert model._score_ws.max_rows == VAECF.SCORE_ROWS == 1024
    s64, n64 = _scores_ref(pr, net, users[:256], rows_dev)
    rec = {}
    rec["full"] = float(((full.double() - s64).abs() / (KAPPA * U_RND * n64)).max())
    c64, cn64 = _scores_ref(pr, net, users, rows_dev)
    c64, cn64 = c64.gather(1, cands), cn64.gather(1, cands)
    rec["cands"] = float(((cand.double() - c64).abs() / (KAPPA * U_RND * cn64)).max())
    # rank: ids are the candidates' item ids as float32
    loader = SimpleNamespace(dataset=SimpleNamespace(data=[[int(u), c] for u, c in zip(pr.users[:4096], cands.cpu().numpy())]))
    got = torch.from_numpy(model.rank(loader)).cuda()
    top = np.argsort(-cand.cpu().numpy(), axis=1, kind="stable")[:, :got.shape[1]]
    rec["rank exact"] = bool(np.array_equal(got.cpu().numpy(), np.take_along_axis(cands.cpu().numpy(), top, 1).astype(np.float32)))
    rec["rank fp64"] = _order_checks(torch.from_numpy(top.copy()).cuda(), cand, c64, KAPPA * U_RND * cn64)[1]
    # full_rank over 26 744 items: seven chunks of the key buffer merged with the running best 50
    fr = []
    for k in (0, 1, 2, 200):
        got = torch.from_numpy(model.full_rank(int(pr.users[k]))).cuda().reshape(1, -1)
        fr.append(_order_checks(got, model._scores(users[k:k + 1]), s64[k:k + 1], KAPPA * U_RND * n64[k:k + 1]))
    rec["full_rank exact"] = all(e for e, _ in fr)
    rec["full_rank fp64"] = all(f for _, f in fr)
    print(f"[vae bench scores] worst error/bound {rec['full']:.3g} (all items), {rec['cands']:.3g} (candidates); {rec}; "
          f"{time.perf_counter() - t0:.1f} s")
    assert rec["full"] <= 1 and rec["cands"] <= 1
    assert all(v for k, v in rec.items() if isinstance(v, bool)), rec
