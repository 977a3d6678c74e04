"""Multi-VAE: one teacher-forced step of drb_vae_train_steps against a float64 reference, on the shared harness (fp64_step.py).

The reference runs the step of csrc/vae.cu (the oracle's network, oracle/vae_oracle.py) on a snapshot of the device's flat
parameter block and optimiser state, with the same host-drawn keep mask and normals, and carries each value's noise scale N
along the chain: a product adds the sum of |contributions|; tanh, exp, log and the softmax carry N through their derivative
and add their own rounding; the row L2 norm, the log-sum-exp over I logits and the bias column sums add one rounding per
term.  There is no discrete part (fp32 throughout, and tanh has no kink): P = 0.

Calibrated on one H100 80GB HBM3 (700 W power limit) over the GPU cases below (dropout on, two hidden layers, odd latent
size, the ragged batch and a user whose item 0 the padding erases): the per-element KAPPA needed under SGD was at most 0.029
(case a; 0.0015 in case b), every Adam step passes at the ladder's lowest rung 0.125; at KAPPA = 0.25 the worst error / bound is 0.40 (Adam) and 0.39
(SGD).  The CPU part runs the same checks with the reference in float32
standing in for the device (rehearsal), and shows that a 1e-3 relative error in the output layer's gradient fails them.
"""
import os
import sys

import numpy as np
import pandas as pd
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fp64_step  # noqa: E402
from fp64_step import F64, Stepper, U_RND, checked_step, report, summary  # noqa: E402
from oracle import vae_oracle as vo  # noqa: E402
from conftest import golden  # noqa: E402

KAPPA = 0.25


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


def vae_ref(net, X, users, I, hidden, lat, dropout, anneal, dt=F64, defects=(), keep=None, eps=None):
    """one train step's gradient, its noise N, the loss and its noise -> harness result (P = 0)"""
    lay, nW = _layers(I, hidden, lat)
    dev = net.device
    W = net.to(dt)
    A = lambda x: x.abs()  # noqa: E731
    half, lo = lat // 2, lat - lat // 2
    R = X[users].to(dt)
    B = R.shape[0]
    nnz = (R != 0).sum(1, keepdim=True).to(dt)
    nrm = R.norm(dim=1, keepdim=True).clamp_min(1e-12)
    x = R / nrm
    if keep is not None:
        x = x * keep.to(dt) * float(np.float32(1.0 / (1.0 - dropout)))
    xN = A(x) * (nnz + 2)

    def wb(L):
        side, k, a, b, wo, bo = lay[L]
        w = W[wo:wo + a * b].view(a, b).T if L == 0 else W[wo:wo + a * b].view(b, a)
        return w, W[bo:bo + b]

    def linear(h, hN, L):
        w, b = wb(L)
        z = h @ w.T + b
        zN = A(h) @ A(w).T + hN @ A(w).T + A(b) + A(z)
        return z, zN

    ne = nd = len(hidden) + 1
    acts = [(x, xN)]
    h, hN = x, xN
    for L in range(ne):
        h, hN = linear(h, hN, L)
        if L < ne - 1:
            a = torch.tanh(h)
            hN = (1 - a * a) * hN + A(a)
            h = a
        acts.append((h, hN))
    mu, muN = h[:, :half], hN[:, :half]
    lv, lvN = h[:, lo:], hN[:, lo:]
    std = torch.exp(0.5 * lv)
    e = torch.zeros_like(mu) if eps is None else eps.to(dev).to(dt)
    z = e * std + mu
    zN = A(e) * std * (0.5 * lvN + 1) + muN + A(z)
    dacts = [(z, zN)]
    h, hN = z, zN
    for l in range(nd):
        h, hN = linear(h, hN, ne + l)
        if l < nd - 1:
            a = torch.tanh(h)
            hN = (1 - a * a) * hN + A(a)
            h = a
        dacts.append((h, hN))
    logit, logitN = dacts[-1]
    lse = torch.logsumexp(logit, 1, keepdim=True)
    p = torch.exp(logit - lse)
    lseN = (p * logitN).sum(1, keepdim=True) + I
    ls = logit - lse
    lsN = logitN + lseN + A(ls)
    rs = R.sum(1, keepdim=True)
    ce_row = (R * ls).sum(1)
    ce_rowN = (A(R) * lsN).sum(1)
    kl_t = 1 + lv - mu * mu - torch.exp(lv)
    kl_row = kl_t.sum(1)
    kl_rowN = (1 + A(lv) + lvN + mu * mu + 2 * A(mu) * muN + torch.exp(lv) * (1 + lvN)).sum(1)
    loss = -ce_row.mean() + (-0.5 * kl_row.mean()) * anneal
    lossN = float(ce_rowN.mean() + 0.5 * anneal * kl_rowN.mean() + A(loss) * 4)
    dz = (p * rs - R) / B
    if "grad_scale" in defects:
        dz = dz * (1 + 1e-3)
    pN = p * (lsN + 1)
    dzN = (pN * A(rs) + p * A(rs) * nnz) / B + A(dz)
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

    cur, curN = dz, dzN
    for l in range(nd - 1, -1, -1):
        L = ne + l
        w, b = wb(L)
        a, aN = dacts[l]
        put(L, cur.T @ a, A(cur).T @ A(a) + curN.T @ A(a) + A(cur).T @ aN, cur.sum(0), (A(cur) + curN).sum(0))
        da = cur @ w
        daN = A(cur) @ A(w) + curN @ A(w) + A(da)
        if l > 0:
            cur, curN = da * (1 - a * a), daN * (1 - a * a) + A(da) * 2 * A(a) * aN + A(da * (1 - a * a))
        else:
            cur, curN = da, daN
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
        a, aN = acts[L]
        gw = cur.T @ a
        put(L, gw, A(cur).T @ A(a) + curN.T @ A(a) + A(cur).T @ aN, cur.sum(0), (A(cur) + curN).sum(0))
        if L > 0:
            w, _ = wb(L)
            da = cur @ w
            daN = A(cur) @ A(w) + curN @ A(w) + A(da)
            cur, curN = da * (1 - a * a), daN * (1 - a * a) + A(da) * 2 * A(a) * aN + A(da * (1 - a * a))
    zero = torch.zeros_like(N)
    return dict(g={"net": g.to(F64)}, N={"net": N}, P={"net": zero}, loss=float(loss), lossN=lossN, lossP=0.0, flagged=0.0)


class _Model:
    phi_max = 0.0
    ladder = True
    ref_uses_kappa = False

    def _model(self, I, hidden, lat, X, dropout, anneal):
        self.I, self.hidden, self.lat, self.dropout, self.anneal = I, list(hidden), lat, dropout, anneal
        self.X = X
        self.kappa = KAPPA

    def reference(self, pre, idx, kappa, dt=F64, defects=(), keep=None, eps=None):
        X = self.X.to(pre["net"].device)
        kp = None if keep is None else keep.to(pre["net"].device)
        return vae_ref(pre["net"], X, idx[0], self.I, self.hidden, self.lat, self.dropout, self.anneal, dt, defects, kp, eps)

    def sections(self):
        lay, _ = _layers(self.I, self.hidden, self.lat)
        out = []
        for side, k, a, b, wo, bo in lay:
            out.append((f"{side}.{2 * k}.weight", "net", wo, wo + a * b, b if (side, k) == ("encoder", 0) else a))
            out.append((f"{side}.{2 * k}.bias", "net", bo, bo + b, 1))
        return out


class VaeGpu(_Model, Stepper):
    device = "cuda"

    def __init__(self, I, hidden, lat, net, X, hist_id, hist_val, users, opt, lr, dropout, anneal_cap):
        from daisyrec_b200 import ops
        self.ops, self.opt, self.lr = ops, opt, lr
        self._model(I, hidden, lat, torch.from_numpy(X), dropout, anneal_cap)
        self.net = torch.from_numpy(np.asarray(net, np.float32)).cuda().contiguous()
        self.t = dict(net=self.net)
        self.planes = (torch.from_numpy(np.asarray(users, np.int64)).cuda(),)
        self.inp = ops.VaeInput(torch.from_numpy(hist_id).cuda(), torch.from_numpy(hist_val).cuda(), I)
        self.hp = ops.hyper(lr, 0.0, 0.0, opt)
        self.ws = ops.VaeWorkspace(I, hidden, lat, opt, self.planes[0].numel(), self.inp.max_row_len, "cuda")
        nW = self.net.numel()
        a = (4 * nW + 255) // 256 * 256
        if opt == "adam":
            f = self.ws.buf[256 + a:256 + 3 * a].view(torch.float32)
            self.mom = {"net": (f[:nW], f[a // 4:a // 4 + nW])}

    def run(self, lo, n, batch, k, adam_step0=0, apply=True, first_step=0, keep=None, eps=None):
        users = self.planes[0][lo:lo + n]
        bits = None
        if keep is not None:
            packed = np.packbits(keep.numpy().reshape(-1).astype(bool), bitorder="little")
            w = np.zeros(self.ops.vae_keep_words(n, self.I) * 4, np.uint8)
            w[:packed.size] = packed
            bits = torch.from_numpy(w.view(np.int32)).cuda()
        out = self.ops.vae_train_steps(self.net, self.ws, self.inp, users, n, 0, 1, self.hp, adam_step0=adam_step0, apply=apply,
                                       training=True, total_anneal_steps=0, anneal_cap=self.anneal, dropout=self.dropout,
                                       keep_bits=bits, eps=eps.cuda().contiguous())
        torch.cuda.synchronize()
        return out.cpu().numpy()


class StandIn(_Model, fp64_step.StandIn):
    def __init__(self, I, hidden, lat, net, X, users, opt, lr, dropout, anneal_cap, defects=()):
        super().__init__(dict(net=net), (users,), opt, lr, 0.0, defects)
        self._model(I, hidden, lat, torch.from_numpy(X), dropout, anneal_cap)

    def stand_in_ref(self, idx, keep=None, eps=None):
        return self.reference(self.t, idx, self.kappa, torch.float32, self.defects, keep, eps)


def _problem(case, opt, dropout):
    """the fixture's synthetic case: initial flat block, dense rule rows, users in the fixture's first-appearance order"""
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
    X = vo.input_rows(g[p + "hist_id"], g[p + "hist_val"], I)
    users = pd.Series(g[p + "df"][0]).unique().astype(np.int64)
    return g, p, I, hidden, lat, net, X, users


def _steps(st, n_rows, batch, dropout, lat, I, n_steps, seed=0):
    torch.manual_seed(seed)
    recs = []
    for s in range(n_steps):
        lo = s * batch
        nb = min(batch, n_rows - lo)
        keep, eps = vo.host_draws(nb, I, lat // 2, dropout)
        recs.append(checked_step(st, lo, nb, batch, f"step {s}", adam_step0=s, keep=keep, eps=eps))
    return recs


# case, optimiser, dropout: (a) one hidden layer, 34 warm users in steps of 16 (the third step is ragged), the user whose item 0
# the padding erases included; (b) two hidden layers, odd latent size 9
CASES = [("a", "sgd", 0.5), ("a", "adam", 0.5), ("b", "sgd", 0.0), ("b", "adam", 0.5)]


@pytest.mark.gpu
@pytest.mark.parametrize("case,opt,dropout", CASES)
def test_teacher_forced_step(case, opt, dropout):
    g, p, I, hidden, lat, net, X, users = _problem(case, opt, dropout)
    hist = (g[p + "hist_id"], g[p + "hist_val"])
    st = VaeGpu(I, hidden, lat, net, X, *hist, users, opt, 0.05 if opt == "sgd" else 0.01, dropout, 0.2)
    recs = _steps(st, len(users), 16, dropout, lat, I, (len(users) + 15) // 16)
    report(f"vae {case} {opt} p={dropout}", recs)
    for r in recs:
        print(summary(r))
    assert all(r["ok"] for r in recs)


@pytest.mark.parametrize("case,opt,dropout", CASES)
def test_rehearsal_on_stand_in(case, opt, dropout):
    """the GPU test body on the float32 reference standing in for the device"""
    g, p, I, hidden, lat, net, X, users = _problem(case, opt, dropout)
    st = StandIn(I, hidden, lat, net, X, users, opt, 0.05 if opt == "sgd" else 0.01, dropout, 0.2)
    recs = _steps(st, len(users), 16, dropout, lat, I, (len(users) + 15) // 16)
    for r in recs:
        print(summary(r))
    assert all(r["ok"] for r in recs)


def test_rehearsal_flags_defective_stand_in():
    g, p, I, hidden, lat, net, X, users = _problem("a", "sgd", 0.5)
    st = StandIn(I, hidden, lat, net, X, users, "sgd", 0.05, 0.5, 0.2, defects=("grad_scale",))
    recs = _steps(st, len(users), 16, 0.5, lat, I, 1)
    print(summary(recs[0]))
    assert not recs[0]["ok"]
