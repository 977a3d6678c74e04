"""The NFM + BPR step (nfm.cu: BatchNorm, the L-layer tower in fp32 and bf16, dropout, the MF dense sweep on the factor
tables) and the FM step (the GEN instantiation of step_kernel.cuh under every loss and optimiser) against float64
references, one teacher-forced step at a time (fp64_step.py: the snapshot, the bound and its checks).  The snapshot also
holds the BatchNorm running statistics; the optimiser state is read from the workspace through mirrors of carve_nfm and of
the MF carve with the bias block.

References.  `nfm_ref`: e = P[u] * Q[item]; BatchNorm with the statistics of each forward call (the positive half and the
negative half separately, biased variance, eps 1e-5) and running statistics (momentum 0.1, unbiased variance, the positive
call first); L x (Linear -> [BN] -> relu | sigmoid | tanh), a dropout factor (fp32 1 / (1 - p)) behind FM_layers and behind
each activation; fm = h + ((u_bias + i_bias) + bias_), pred = <fm, wp>; BPR with gamma = 1e-10; the un-squared L1 / Frobenius
regulariser on the factor rows counted per occurrence; the closed-form BatchNorm backward.  With tower_dtype 1 both operands
of each layer's three GEMMs are rounded to bf16: h_in and W (forward), h_prev and dz (weight gradient), dz and W (input
gradient).  `nfm_scores_ref`: the same forward in eval mode on the running statistics.  `fm_ref`: <p, q> + ((u_bias + i_bias)
+ bias_), the five losses with pair_loss's coefficients (HL passes the gradient at equality; CL / SL take the label plane in
place of the negative and touch no j row), the MF regulariser on P and Q and none on the biases.

N_e: BatchNorm's backward is expanded as |B dxh| + |sum dxh| + |xhat| |sum dxh xhat| (times inv_std / B) and its centring as
|x| + |mean|, so the cancellation inside BatchNorm and the inv_std gain show up in N_e.  P_e: relu gates within their noise
of 0, HL margins within their noise of 0, bf16 operands within their noise of a rounding midpoint.  A Linear bias in front of
a BatchNorm, and BN0's beta when a Linear follows it, have a mathematically zero gradient: their interval contains 0, so the
Adam bound is about lr there by construction.

Exact: under BPR the u_bias slots and bias_ are bit-identical after every step (their gradient is exactly 0: per triple the
two halves cancel); under SGD untouched rows and i_bias slots are bit-identical; the gradient accumulators and row counters
are zero after every applied step; apply = 0 leaves P, Q, bias and the network block alone (NFM's running statistics move).
"""
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fp64_step  # noqa: E402
from fp64_step import (F64, GAMMA, U_RND, Flags, Stepper, _A, br, carve, checked_step, device_tensor,  # noqa: E402
                       launch_vs_singles, mm, opt_apply, report, rnd, summary, views)

# Calibrated on one H100 80GB HBM3 (700 W power limit) over every GPU case below; the GPU part of the file runs in 32 s there.
# "Needed" is the per-element KAPPA of an SGD step where P_e = 0, else (Adam, Adagrad, RMSprop, bf16) the smallest KAPPA of
# KAPPA_LADDER at which every element of the step passes; the ladder starts at 0.125.
#   NFM fp32: 1.0 (geometry F = 6, L = 3, sigmoid; 0.35 on the launches, <= 0.125 at the bench shape), hence 2.
#   NFM bf16: 1.0 (the launches; <= 0.5 elsewhere), hence 2.
#   NFM with dropout_engine 'philox' (test_nfm_philox_dropout, p = 0.5, the hook's masks): fp32 0.005, worst error/bound
#     0.49; bf16 0.5 (ladder), worst error/bound 1.00, at most 33 % of the intermediates flagged.
#   FM: 1.94 (HL under SGD, P[2223, 44]; 1.69 at the bench shape under SGD), hence 4.
# Power (test_harness_power_in_every_gpu_configuration): in every (bn, L, act) a GPU case runs, a 1e-3 relative gradient error
# (5e-3 in bf16) in P, W0, wp or BN0's gamma and each bf16 operand left unrounded exceed the bound.  The defective stand-ins
# are caught at 3.2e3 - 5e7 x the bound (test_harness_flags_defective_stand_in prints each ratio).
KAPPA = {"nfm": 2.0, "nfm_bf16": 2.0, "fm": 4.0}
# The share of rounded or gated intermediates of a step flagged as possible midpoint / gate flips: at most 0.47 measured (bf16
# launches, BatchNorm, L = 1; 0.33 at the bench shape), hence the 0.6 ceiling.
PHI_MAX = 0.6
ACTS = ("relu", "sigmoid", "tanh")
OPTS = ("sgd", "adam", "adagrad", "rmsprop")
FM_LOSSES = ("BPR", "CL", "SL", "HL", "TL")


def kappa_of(model, td=0):
    return KAPPA["nfm_bf16"] if model == "nfm" and td == 1 else KAPPA[model]


def _Z(t):
    return torch.zeros(t.shape, dtype=F64, device=t.device)


# ---------------------------------------------------------------- layouts
def nfm_layout(F, L, bn):
    """the flat network block in module-registration order: name -> (lo, hi)"""
    lay, o = {}, 0
    if bn:
        lay["bn0.g"], lay["bn0.b"] = (0, F), (F, 2 * F)
        o = 2 * F
    for l in range(L):
        lay[f"W{l}"], lay[f"b{l}"] = (o, o + F * F), (o + F * F, o + F * F + F)
        o += F * F + F
        if bn:
            lay[f"bn{l + 1}.g"], lay[f"bn{l + 1}.b"] = (o, o + F), (o + F, o + 2 * F)
            o += 2 * F
    lay["wp"] = (o, o + F)
    return lay, o + F


def nfm_ws_layout(U, I, F, L, bn, opt, max_rows):
    """mirror of carve_nfm (nfm.cu): name -> (byte offset, bytes), total"""
    nN, nb, act = nfm_layout(F, L, bn)[1], U + I + 1, 4 * max_rows * F
    parts = [("hdr", 256), ("gP", 4 * U * F), ("gQ", 4 * I * F), ("gB", 4 * nb), ("gN", 4 * nN), ("cntU", 4 * U), ("cntI", 8 * I)]
    if opt == "adam":
        parts += [("mP", 4 * U * F), ("vP", 4 * U * F), ("mQ", 4 * I * F), ("vQ", 4 * I * F), ("mB", 4 * nb), ("vB", 4 * nb),
                  ("mN", 4 * nN), ("vN", 4 * nN)]
    parts += [("stats", 8 * 2 * 4 * F), ("bnm", 4 * (1 + L) * 2 * 2 * F), ("scratch", 64), ("pred", 4 * max_rows),
              ("coef", 4 * max_rows), ("e", act), ("xh0", act), ("h0", act)]
    for l in range(L):
        parts += [(f"zpre{l}", act), (f"xh{l}", act), (f"z{l}", act), (f"h{l}", act)]
    parts += [("fm", act), ("dh", act), ("tmp", act)]
    return carve(parts)


def fm_ws_layout(U, I, F, opt):
    """mirror of carve (step.cuh) with the bias block (fm = 1)"""
    nb = U + I + 1
    parts = [("hdr", 256), ("gP", 4 * U * F), ("gQ", 4 * I * F), ("cntU", 4 * U), ("cntI", 8 * I)]
    if opt != "sgd":
        parts += [("mP", 4 * U * F)] + ([("vP", 4 * U * F)] if opt == "adam" else [])
        parts += [("mQ", 4 * I * F)] + ([("vQ", 4 * I * F)] if opt == "adam" else [])
    parts += [("gB", 4 * nb)] + ([("mB", 4 * nb)] if opt != "sgd" else []) + ([("vB", 4 * nb)] if opt == "adam" else [])
    return carve(parts)


# ---------------------------------------------------------------- shared pieces
def row_reg(T, idx_list, reg):
    """un-squared L1 / Frobenius regulariser of the rows T[idx] per index plane, counted per occurrence -> (g, N, loss, lossN)"""
    reg1, reg2 = reg
    g, N = _Z(T), _Z(T)
    if not (reg1 or reg2):
        return g, N, 0.0, 0.0
    src = T.to(F64)
    loss = lossN = 0.0
    for idx in idx_list:
        rows = src[idx]
        l1, nr = float(rows.abs().sum()), math.sqrt(float((rows ** 2).sum()))
        inv = float(np.float32(1.0 / nr)) if nr > 0 else 0.0
        t = reg1 * torch.sign(rows) + reg2 * rows * inv
        g.index_add_(0, idx, t)
        N.index_add_(0, idx, t.abs())
        loss += reg1 * l1 + reg2 * nr
        lossN += abs(reg1 * l1) + abs(reg2 * nr)
    return g, N, loss, lossN


def keep_factors(keep_bytes, L, B, F, p, dt=F64):
    """device keep bytes of one step [2][1 + L][B][F] -> factor tensors [1 + L, 2B, F] (the kernel's fp32 1 / (1 - p))"""
    scale = float(np.float32(1.0) / np.float32(1.0 - p))
    k = keep_bytes.reshape(2, 1 + L, B, F).to(dt) * scale
    return torch.cat([k[0], k[1]], 1)


# ---------------------------------------------------------------- NFM reference
def _bn_fwd(x, xN, xP, gam, bet, G, ku):
    """BatchNorm (train) over G row groups of x [R, F] -> dict of the pieces the backward and the running statistics need"""
    R, F = x.shape
    xv, xNv, xPv = x.view(G, -1, F), xN.view(G, -1, F), xP.view(G, -1, F)
    n = xv.shape[1]
    mean = xv.mean(1, keepdim=True)
    c = xv - mean
    var = (c * c).mean(1, keepdim=True)
    inv = 1.0 / torch.sqrt(var + 1e-5)
    xh = c * inv
    y = xh * gam + bet
    xhA, invA, cA = _A(xh), _A(inv), _A(c)
    # Sums over the n rows of a half add n independent per-row errors (roundings, atomics order): they add in quadrature
    # (qmean).  Adding them as absolute values would compound by ~sqrt(n) at every BatchNorm and leave the bound of a deep
    # BatchNorm tower orders of magnitude above any real error.  The parts of xhat's error that are common to a whole column
    # -- the fp32 rounding of the mean (a shift) and the noise of inv_std (a scale) -- are kept apart and enter the
    # backward's sums with the sign-aware column sums |sum dxh| and |sum dxh xhat| instead.
    qmean = lambda d: torch.sqrt((d * d).sum(1, keepdim=True)) / n
    cN = xNv + qmean(xNv)                                                # the variance pass runs in fp64: input noise only
    cP = xPv + qmean(xPv)
    varN = 2 * qmean(cA * cN) + _A(var)
    varP = 2 * qmean(cA * cP)
    den = _A(var) + 1e-5
    rel_inv = 0.5 * varN / den + 2.0                                     # relative noise of inv_std, in units of u
    rel_invP = 0.5 * varP / den
    pert = lambda d: invA * (d + qmean(d) + xhA * qmean(xhA * d))
    xh_ind = pert(xNv) + invA * cA + xhA                                 # per row: input noise, x - mean, the product
    shift = invA * _A(mean)                                              # per column: the fp32 mean, centring |x| + |mean|
    xhN = xh_ind + shift + xhA * rel_inv
    xhP = pert(xPv) + xhA * rel_invP
    gA = _A(gam)
    yN = xhN * gA + _A(xh * gam) + _A(bet) + _A(y)
    yP = xhP * gA
    ssum = (c * c).sum(1)                                                # [G, F]
    return dict(y=y.reshape(R, F), yN=yN.reshape(R, F), yP=yP.reshape(R, F), xh=xh, xhN=xhN, xhP=xhP, inv=inv, n=n, G=G,
                mean=mean[:, 0], ss=ssum, meanN=(xNv.mean(1) + _A(mean[:, 0])), meanP=xPv.mean(1),
                varN=varN[:, 0], varP=varP[:, 0], rel_inv=rel_inv, rel_invP=rel_invP, xh_ind=xh_ind, shift=shift)


def _bn_running(b, rm, rv, defects):
    """momentum 0.1, unbiased variance, the positive call first -> (mean, var, meanN, varN, meanP, varP) float64"""
    rm, rv = rm.to(F64), rv.to(F64)
    n = b["n"]
    order = list(range(b["G"]))
    if b["G"] == 1:
        order = [0, 0]
    elif "neg_running_first" in defects:
        order = [1, 0]
    mN, vN, mP, vP = _Z(rm), _Z(rv), _Z(rm), _Z(rv)
    for h in order:
        var = b["ss"][h].to(F64) / (n if "biased_running_var" in defects else max(n - 1, 1))
        rm = 0.9 * rm + 0.1 * b["mean"][h].to(F64)
        rv = 0.9 * rv + 0.1 * var
        mN, vN = 0.9 * mN + 0.1 * b["meanN"][h], 0.9 * vN + 0.1 * b["varN"][h] * n / max(n - 1, 1)
        mP, vP = 0.9 * mP + 0.1 * b["meanP"][h], 0.9 * vP + 0.1 * b["varP"][h] * n / max(n - 1, 1)
    return rm, rv, mN, vN, mP, vP


def _act(act, z, zN, zP, st, ku):
    if act == 0:
        unc = _A(z) <= ku * zN + zP
        st.add(unc)
        on = (z > 0) | unc
        return torch.where(z > 0, z, torch.zeros_like(z)), torch.where(on, zN, 0.0), torch.where(on, zP, 0.0), unc
    h = torch.sigmoid(z) if act == 1 else torch.tanh(z)
    d = _A(h * (1 - h)) if act == 1 else _A(1 - h * h)
    return h, d * zN + _A(h), d * zP, None


def _forward(P, Q, bias, N, Rs, U, I, L, bn, act, users, items, B, td, keep, dt, defects, st, train):
    """the NFM forward on rows (users[r], items[r]); train: BatchNorm on the statistics of each half of B rows"""
    F = P.shape[1]
    ku = st.k * U_RND
    lay, _ = nfm_layout(F, L, bn)
    Nd = N.to(dt)
    sec = lambda k: Nd[lay[k][0]:lay[k][1]]
    bf = td == 1
    rnd_on = lambda op, l: bf and not (f"unrounded_{op}" in defects and l == 0)
    pu, qit = P.to(dt)[users], Q.to(dt)[items]
    e = pu * qit
    h, hN, hP = e, _A(e), _Z(e)
    G = 1 if "bn_all_rows" in defects else 2
    bns, layers = [], []

    def bn_apply(x, xN, xP, k, gname):
        gam, bet = sec(f"{gname}.g"), sec(f"{gname}.b")
        if train:
            b = _bn_fwd(x, xN, xP, gam, bet, G, ku)
            bns.append(b)
            return b["y"], b["yN"], b["yP"], b
        rm, rv = Rs.to(dt)[k * 2 * F:k * 2 * F + F], Rs.to(dt)[k * 2 * F + F:(k + 1) * 2 * F]
        inv = 1.0 / torch.sqrt(rv + 1e-5)
        xh = (x - rm) * inv
        y = xh * gam + bet
        xhN = (xN + _A(x) + _A(rm)) * _A(inv) + 2 * _A(xh)
        return y, xhN * _A(gam) + _A(xh * gam) + _A(bet) + _A(y), xP * _A(inv * gam), None

    if bn:
        h, hN, hP, _ = bn_apply(h, hN, hP, 0, "bn0")
    if keep is not None:
        k0 = keep[0]
        h, hN, hP = h * k0, hN * k0 + _A(h * k0), hP * k0
    hin = (h, hN, hP)
    for l in range(L):
        W, b = sec(f"W{l}").view(F, F), sec(f"b{l}")
        a = rnd(*hin, st, rnd_on("h", l))
        Wr = br(W) if rnd_on("W", l) else W
        zv, zN, zP = mm(*a, Wr, _Z(Wr), _Z(Wr), True)
        z = zv + b
        zN = zN + _A(b) + _A(z)
        bnl = None
        if bn:
            z, zN, zP, bnl = bn_apply(z, zN, zP, 1 + l, f"bn{l + 1}")
        hh, hhN, hhP, unc = _act(act, z, zN, zP, st, ku)
        layers.append(dict(hin=hin, z=z, zN=zN, zP=zP, h=hh, unc=unc, bn=bnl, W=W, b=b))
        if keep is not None:
            kl = keep[1 + l]
            hh, hhN, hhP = hh * kl, hhN * kl + _A(hh * kl), hhP * kl
        hin = (hh, hhN, hhP)
    h, hN, hP = hin
    bd = bias.to(dt)
    ub, ib, b0 = bd[users], bd[U + items], bd[U + I]
    bsum = (ub + ib) + b0
    fm = h + bsum[:, None]
    fmN = hN + (_A(ub) + _A(ib) + _A(b0) + _A(ub + ib) + _A(bsum))[:, None] + _A(fm)
    fmP = hP
    wp = sec("wp")
    pred = fm @ wp
    predN = fmN @ _A(wp) + _A(fm) @ _A(wp)
    predP = fmP @ _A(wp)
    return dict(pu=pu, qit=qit, fm=fm, fmN=fmN, fmP=fmP, pred=pred, predN=predN, predP=predP, wp=wp, layers=layers, bns=bns,
                lay=lay, sec=sec, rnd_on=rnd_on, bsum=bsum)


def _bn_bwd(b, dz, dzN, dzP, gam):
    """closed-form BatchNorm backward -> (dx, N, P, ggamma, N, P, gbeta, N, P)"""
    G, n = b["G"], b["n"]
    F = dz.shape[1]
    dzv, dzNv, dzPv = dz.view(G, n, F), dzN.view(G, n, F), dzP.view(G, n, F)
    xh, xhN, xhP = b["xh"], b["xhN"], b["xhP"]
    xhA = _A(xh)
    gg = (dzv * xh).sum((0, 1))
    ggN = (dzNv * xhA + _A(dzv) * xhN + _A(dzv * xh)).sum((0, 1))
    ggP = (dzPv * xhA + _A(dzv) * xhP).sum((0, 1))
    gb, gbN, gbP = dzv.sum((0, 1)), (dzNv + _A(dzv)).sum((0, 1)), dzPv.sum((0, 1))
    gA = _A(gam)
    dxh = dzv * gam
    dxhN, dxhP = dzNv * gA, dzPv * gA
    # nfm_bn_bwd_kernel forms dxh, the column sums and the cancellation B dxh - sum dxh - xhat sum(dxh xhat) in fp64 and rounds
    # dx once: the expansion |B dxh| + |sum dxh| + |xhat| |sum dxh xhat| enters through the noise of its fp32 inputs only
    S1, S2 = dxh.to(F64).sum(1, keepdim=True), (dxh.to(F64) * xh.to(F64)).sum(1, keepdim=True)
    inv = b["inv"]
    dx = (inv.to(F64) / n * (n * dxh.to(F64) - S1 - xh.to(F64) * S2)).to(dz.dtype)
    s = _A(inv) / n
    S2A = _A(S2)
    qsum = lambda d: torch.sqrt((d * d).sum(1, keepdim=True))           # independent per-row errors, see _bn_fwd
    S2N = qsum(dxhN * xhA + _A(dxh) * b["xh_ind"]) + b["shift"] * _A(S1) + b["rel_inv"] * S2A
    dxN = s * (n * dxhN + qsum(dxhN) + xhA * S2N + xhN * S2A) + _A(dx) * (1 + b["rel_inv"])
    dxP = s * (n * dxhP + qsum(dxhP) + xhA * qsum(dxhP * xhA + _A(dxh) * xhP) + xhP * S2A) + _A(dx) * b["rel_invP"]
    R = G * n
    return dx.reshape(R, F), dxN.reshape(R, F), dxP.reshape(R, F), gg, ggN, ggP, gb, gbN, gbP


def nfm_ref(P, Q, bias, N, Rs, U, I, L, bn, act, bu, bi, bj, reg=(0.0, 0.0), td=0, keep=None, dt=F64, defects=(),
            kappa=None):
    """one NFM + BPR step (gradients, not applied) -> dict(g, N, P: {"P", "Q", "bias", "N"}, Rs, RsN, RsP, loss, lossN, lossP,
    flagged).  keep: dropout factors [1 + L, 2B, F] or None."""
    st = Flags(kappa_of("nfm", td) if kappa is None else kappa)
    ku = st.k * U_RND
    dev, F, B = P.device, P.shape[1], bu.numel()
    users, items = torch.cat([bu, bu]), torch.cat([bi, bj])
    f = _forward(P, Q, bias, N, Rs, U, I, L, bn, act, users, items, B, td, keep, dt, defects, st, True)
    lay, sec, rnd_on = f["lay"], f["sec"], f["rnd_on"]
    nN = nfm_layout(F, L, bn)[1]
    pred, predN, predP = f["pred"], f["predN"], f["predP"]
    x = pred[:B] - pred[B:]
    xN = predN[:B] + predN[B:] + _A(x)
    xP = predP[:B] + predP[B:]
    s = 1.0 / (1.0 + torch.exp(-x))
    c = -(s * (1.0 - s)) / (GAMMA + s)
    lt = -torch.log(GAMMA + s)
    cN, cP = xN / 4 + _A(c), xP / 4
    cr, crN, crP = torch.cat([c, -c]), torch.cat([cN, cN]), torch.cat([cP, cP])
    # head backward
    wp, fm, fmN, fmP = f["wp"], f["fm"], f["fmN"], f["fmP"]
    wA = _A(wp)
    dh = cr[:, None] * wp[None, :]
    dhN, dhP = crN[:, None] * wA + _A(dh), crP[:, None] * wA
    gN, NN, PN = torch.zeros(nN, dtype=F64, device=dev), torch.zeros(nN, dtype=F64, device=dev), torch.zeros(nN, dtype=F64, device=dev)

    def put(name, g_, n_, p_):
        lo, hi = lay[name]
        gN[lo:hi] += g_.to(F64).reshape(-1); NN[lo:hi] += n_.reshape(-1); PN[lo:hi] += p_.reshape(-1)

    put("wp", (cr[:, None] * fm).sum(0), (crN[:, None] * _A(fm) + _A(cr)[:, None] * fmN + _A(cr[:, None] * fm)).sum(0),
        (crP[:, None] * _A(fm) + _A(cr)[:, None] * fmP).sum(0))
    bs = dh.sum(1)
    bsN, bsP = dhN.sum(1) + _A(bs), dhP.sum(1)
    gB, NB, PB = (torch.zeros(U + I + 1, dtype=F64, device=dev) for _ in range(3))
    gB.index_add_(0, U + items, bs.to(F64)); NB.index_add_(0, U + items, bsN); PB.index_add_(0, U + items, bsP)
    if "ubias_per_half" in defects:                 # the user / global terms summed per half instead of per triple
        gu = torch.zeros(U + I + 1, dtype=dt, device=dev)
        gu.index_add_(0, bu, bs[:B]); gu.index_add_(0, bu, bs[B:])
        gu[U + I] = bs[:B].sum() + bs[B:].sum()
        gB[:U] += gu[:U].to(F64); gB[U + I] += gu[U + I].to(F64)
    # tower backward
    for l in reversed(range(L)):
        a = f["layers"][l]
        if keep is not None:
            kl = keep[1 + l]
            dh, dhN, dhP = dh * kl, dhN * kl + _A(dh * kl), dhP * kl
        z, zN, zP, h = a["z"], a["zN"], a["zP"], a["h"]
        if act == 0:
            gate = (z > 0).to(dt)
            dz = dh * gate
            dzN = torch.where(a["unc"], 0.0, dhN * gate)
            dzP = torch.where(a["unc"], _A(dh) + ku * dhN + dhP, dhP * gate)
        else:
            if act == 1:
                d = z * (1 - z) if "sigmoid_from_z" in defects else h * (1 - h)
                dd = _A(1 - 2 * h) * _A(h * (1 - h))
            else:
                d, dd = 1 - h * h, 2 * _A(h) * _A(1 - h * h)
            dz = dh * d
            dzN = dhN * _A(d) + _A(dh) * (dd * zN + _A(d) + _A(h)) + _A(dz)
            dzP = dhP * _A(d) + _A(dh) * dd * zP
        if bn:
            gam = sec(f"bn{l + 1}.g")
            dz, dzN, dzP, gg, ggN, ggP, gbt, gbtN, gbtP = _bn_bwd(a["bn"], dz, dzN, dzP, gam)
            put(f"bn{l + 1}.g", gg, ggN, ggP)
            put(f"bn{l + 1}.b", gbt, gbtN, gbtP)
            dzN = dzN + _A(dz)
        put(f"b{l}", dz.sum(0), (dzN + _A(dz)).sum(0), dzP.sum(0))
        hp_w = rnd(*a["hin"], Flags(st.k), rnd_on("hprev", l))
        dz_w = rnd(dz, dzN, dzP, st, rnd_on("dz", l))
        v, n_, p_ = mm(dz_w[0].T.contiguous(), dz_w[1].T.contiguous(), dz_w[2].T.contiguous(), *hp_w, False)
        put(f"W{l}", v, n_, p_)
        dz_i = rnd(dz, dzN, dzP, Flags(st.k), rnd_on("dzi", l))
        Wi = br(a["W"]) if rnd_on("Wi", l) else a["W"]
        dh, dhN, dhP = mm(*dz_i, Wi, _Z(Wi), _Z(Wi), False)
        dhN = dhN + _A(dh)
    if keep is not None:
        k0 = keep[0]
        dh, dhN, dhP = dh * k0, dhN * k0 + _A(dh * k0), dhP * k0
    if bn:
        dh, dhN, dhP, gg, ggN, ggP, gbt, gbtN, gbtP = _bn_bwd(f["bns"][0], dh, dhN, dhP, sec("bn0.g"))
        put("bn0.g", gg, ggN, ggP)
        put("bn0.b", gbt, gbtN, gbtP)
        dhN = dhN + _A(dh)
    pu, qit = f["pu"], f["qit"]
    gT = {}
    for name, idx, other, n_tab in (("P", users, qit, U), ("Q", items, pu, I)):
        g_ = torch.zeros(n_tab, F, dtype=F64, device=dev)
        N_, P_ = torch.zeros_like(g_), torch.zeros_like(g_)
        g_.index_add_(0, idx, (dh * other).to(F64))
        N_.index_add_(0, idx, dhN * _A(other) + _A(dh * other))
        P_.index_add_(0, idx, dhP * _A(other))
        gT[name] = [g_, N_, P_]
    gr, grN, lreg, lregN = row_reg(torch.cat([P, Q]), (bu, U + bi, U + bj), reg)
    for name, sl in (("P", slice(0, U)), ("Q", slice(U, U + I))):
        gT[name][0] = gT[name][0] + gr[sl]
        gT[name][1] = gT[name][1] + grN[sl] + _A(gT[name][0])
    NB = NB + _A(gB)
    NN = NN + _A(gN)
    # running statistics
    Rn, RN, RP = None, None, None
    if bn:
        parts = [_bn_running(b, Rs[k * 2 * F:k * 2 * F + F], Rs[k * 2 * F + F:(k + 1) * 2 * F], defects) for k, b in enumerate(f["bns"])]
        Rn = torch.cat([torch.cat([p_[0], p_[1]]) for p_ in parts])
        RN = torch.cat([torch.cat([p_[2], p_[3]]) for p_ in parts])
        RP = torch.cat([torch.cat([p_[4], p_[5]]) for p_ in parts])
    loss = float(lt.to(F64).sum()) + lreg
    return dict(g=dict(P=gT["P"][0], Q=gT["Q"][0], bias=gB, N=gN), N=dict(P=gT["P"][1], Q=gT["Q"][1], bias=NB, N=NN),
                P=dict(P=gT["P"][2], Q=gT["Q"][2], bias=PB, N=PN), Rs=Rn, RsN=RN, RsP=RP, loss=loss,
                lossN=float((xN + _A(lt)).sum()) + lregN + abs(loss), lossP=float(xP.sum()), flagged=st.frac())


def nfm_scores_ref(P, Q, bias, N, Rs, U, I, L, bn, act, u, i, td=0, kappa=None):
    """eval-mode scores of the pairs (u[k], i[k]) -> (value, N, P)"""
    st = Flags(kappa_of("nfm", td) if kappa is None else kappa)
    f = _forward(P, Q, bias, N, Rs, U, I, L, bn, act, u, i, u.numel(), td, None, F64, (), st, False)
    return f["pred"], f["predN"], f["predP"]


# ---------------------------------------------------------------- FM reference
def fm_ref(P, Q, bias, U, I, bu, bi, bj, loss, reg=(0.0, 0.0), dt=F64, defects=(), kappa=None):
    """one FM step (gradients, not applied) -> dict(g, N, P: {"P", "Q", "bias"}, loss, lossN, lossP, flagged)"""
    k = KAPPA["fm"] if kappa is None else kappa
    ku = k * U_RND
    dev, F = P.device, P.shape[1]
    pw = loss in ("CL", "SL")
    Pd, Qd, bd = P.to(dt), Q.to(dt), bias.to(dt)
    p, qi = Pd[bu], Qd[bi]
    ub, ib, b0 = bd[bu], bd[U + bi], bd[U + I]
    bterm = lambda u_, i_: (_A(u_) + _A(i_) + _A(b0) + _A(u_ + i_) + _A((u_ + i_) + b0))
    pos = (p * qi).sum(1) + ((ub + ib) + b0)
    posN = (_A(p) * _A(qi)).sum(1) + bterm(ub, ib) + _A(pos)
    scatter_j = not pw or "label_scatter" in defects
    if not pw:
        qj, jb = Qd[bj], bd[U + bj]
        neg = (p * qj).sum(1) + ((ub + jb) + b0)
        negN = (_A(p) * _A(qj)).sum(1) + bterm(ub, jb) + _A(neg)
    else:
        qj = Qd[bj] if "label_scatter" in defects else torch.zeros_like(p)
        neg, negN = bj.to(dt), torch.zeros(bu.numel(), dtype=F64, device=dev)
    zero = torch.zeros_like(pos)
    cP = cnP = torch.zeros(bu.numel(), dtype=F64, device=dev)
    flagged = 0.0
    if loss == "BPR":
        x = pos - neg
        s = 1.0 / (1.0 + torch.exp(-x))
        c = -(s * (1.0 - s)) / (GAMMA + s)
        cn, lt = -c, -torch.log(GAMMA + s)
        cN = (posN + negN) / 4 + _A(c)
        cnN = cN
    elif loss == "CL":
        z = torch.exp(-pos.abs())
        dls = torch.where(pos < 0, 1 - z / (1 + z), z / (1 + z))
        c, cn = (1 - neg) - dls, zero
        lt = (1 - neg) * pos - (torch.clamp(pos, max=0) - torch.log1p(z))
        cN, cnN = posN / 4 + _A(1 - neg) + _A(dls) + _A(c), _Z(c)
    elif loss == "SL":
        d = pos - neg
        c, cn, lt = 2 * d, zero, d * d
        cN, cnN = 2 * (posN + _A(neg) + _A(d)) + _A(c), _Z(c)
    elif loss == "HL":
        m = 1 - (pos - neg)
        unc = _A(m) <= ku * (posN + negN + 1 + _A(pos - neg))
        flagged = float(unc.to(F64).mean())
        on = (m > 0) if "hl_cut" in defects else (m >= 0)
        c = torch.where(on, -1.0, 0.0).to(dt)
        cn, lt = -c, torch.clamp(m, min=0)
        cN, cnN = _Z(c), _Z(c)
        cP = cnP = unc.to(F64)
    else:                                            # TL
        s1, s2 = torch.sigmoid(neg - pos), torch.sigmoid(neg * neg)
        c = -(s1 * (1 - s1))
        cn = s1 * (1 - s1) + s2 * (1 - s2) * 2 * neg
        lt = s1 + s2
        cN = 0.1 * (posN + negN) + _A(c)
        cnN = 0.1 * posN + (0.6 + 0.4 * _A(neg * neg)) * negN + _A(cn) + _A(s1 * (1 - s1)) + _A(s2 * (1 - s2) * 2 * neg)
    cA, cnA = _A(c)[:, None], _A(cn)[:, None]
    qiA, qjA, pA = _A(qi), _A(qj), _A(p)
    if loss == "BPR":
        gu = c[:, None] * (qi - qj)
        guN = cA * (qiA + qjA) * 2 + cN[:, None] * (qiA + qjA) + _A(gu)
    else:
        gu = c[:, None] * qi + cn[:, None] * qj
        guN = cA * qiA + cnA * qjA + cN[:, None] * qiA + cnN[:, None] * qjA + _A(gu)
    guP = cP[:, None] * qiA + cnP[:, None] * qjA
    gi, gj = c[:, None] * p, cn[:, None] * p
    gP, NP, PP = torch.zeros(U, F, dtype=F64, device=dev), torch.zeros(U, F, dtype=F64, device=dev), torch.zeros(U, F, dtype=F64, device=dev)
    gQ, NQ, PQ = torch.zeros(I, F, dtype=F64, device=dev), torch.zeros(I, F, dtype=F64, device=dev), torch.zeros(I, F, dtype=F64, device=dev)
    gP.index_add_(0, bu, gu.to(F64)); NP.index_add_(0, bu, guN); PP.index_add_(0, bu, guP)
    gQ.index_add_(0, bi, gi.to(F64)); NQ.index_add_(0, bi, cN[:, None] * pA + _A(gi)); PQ.index_add_(0, bi, cP[:, None] * pA)
    if not pw:
        gQ.index_add_(0, bj, gj.to(F64)); NQ.index_add_(0, bj, cnN[:, None] * pA + _A(gj)); PQ.index_add_(0, bj, cnP[:, None] * pA)
    gB, NB, PB = (torch.zeros(U + I + 1, dtype=F64, device=dev) for _ in range(3))
    both = c if pw else c + cn                       # BPR: c + (-c) == 0 exactly
    bothN = cN if pw else (cN + cnN + _A(both)) * (loss != "BPR")
    bothP = cP if pw else (cP + cnP) * (loss != "BPR")
    gB.index_add_(0, bu, both.to(F64)); NB.index_add_(0, bu, bothN); PB.index_add_(0, bu, bothP)
    gB.index_add_(0, U + bi, c.to(F64)); NB.index_add_(0, U + bi, cN); PB.index_add_(0, U + bi, cP)
    if not pw:
        gB.index_add_(0, U + bj, cn.to(F64)); NB.index_add_(0, U + bj, cnN); PB.index_add_(0, U + bj, cnP)
    gB[U + I] = both.to(F64).sum(); NB[U + I] = bothN.sum(); PB[U + I] = bothP.sum()
    NB = NB + _A(gB)
    planes = (bu, U + bi) + ((U + bj,) if scatter_j else ())
    gr, grN, lreg, lregN = row_reg(torch.cat([P, Q]), planes, reg)
    gP, gQ = gP + gr[:U], gQ + gr[U:]
    NP, NQ = NP + grN[:U] + _A(gP), NQ + grN[U:] + _A(gQ)
    lval = float(lt.to(F64).sum()) + lreg
    lN = float(((posN + negN) + _A(lt)).sum()) + lregN + abs(lval)
    return dict(g=dict(P=gP, Q=gQ, bias=gB), N=dict(P=NP, Q=NQ, bias=NB), P=dict(P=PP, Q=PQ, bias=PB), loss=lval, lossN=lN,
                lossP=float((cP + cnP).sum()), flagged=flagged)


# ---------------------------------------------------------------- steppers: the device and its CPU stand-in
def _rs_ratio(res, got):
    if res.get("Rs") is None:
        return 0.0
    want = res["Rs"]
    err = (got.to(F64) - want).abs()
    bound = KAPPA["nfm"] * U_RND * res["RsN"] + res["RsP"] + 4 * U_RND * want.abs() + 1e-30
    return float((err / bound).max())


class _Model:
    """NFM (model "nfm") or FM on P, Q, bias (and the network block N, the running statistics Rs): the reference call, the
    compared sections and the exact checks"""
    phi_max = PHI_MAX
    L = bn = act = td = 0
    loss, dropout = "BPR", 0.0

    def _model(self, model, U, I, F):
        self.model, self.U, self.I, self.F = model, U, I, F
        self.kappa = kappa_of(model, self.td)

    def reference(self, pre, idx, kappa, dt=F64, defects=(), keep=None):
        if self.model == "fm":
            return fm_ref(pre["P"], pre["Q"], pre["bias"], self.U, self.I, *idx, self.loss, self.reg, dt, defects, kappa)
        kf = None if keep is None else keep_factors(keep.to(pre["P"].device), self.L, idx[0].numel(), self.F, self.dropout, dt)
        return nfm_ref(pre["P"], pre["Q"], pre["bias"], pre["N"], pre["Rs"], self.U, self.I, self.L, self.bn, self.act, *idx,
                       self.reg, self.td, kf, dt, defects, kappa)

    def sections(self):
        U, I, F = self.U, self.I, self.F
        out = [("P", "P", 0, U * F, F), ("Q", "Q", 0, I * F, F), ("u_bias", "bias", 0, U, 1), ("i_bias", "bias", U, U + I, 1),
               ("bias_", "bias", U + I, U + I + 1, 1)]
        if self.model == "nfm":
            out += [(k, "N", a, b, 1) for k, (a, b) in nfm_layout(F, self.L, self.bn)[0].items()]
        return out

    def checks(self, pre, post, res, apply):
        out = dict(rs_ratio=_rs_ratio(res, post["Rs"]) if "Rs" in post else 0.0)
        if apply:
            # BPR: the user and global bias slots are bit-identical (their gradient is exactly 0); every accumulator is clean
            U, I = self.U, self.I
            out["bias_exact"] = not (self.model == "nfm" or self.loss == "BPR") or bool(
                torch.equal(pre["bias"][:U], post["bias"][:U]) and torch.equal(pre["bias"][U + I:], post["bias"][U + I:]))
            out["clean"] = self.clean()
        return out


class _Gpu(_Model, Stepper):
    device = "cuda"

    def _workspace(self, buf, lay, keys):
        """views of the accumulators and counters, and of the optimiser state of each parameter tensor"""
        acc = [k for k in ("gP", "gQ", "gB", "gN") if k in lay]
        self.acc = views(buf, lay, dict({k: torch.float32 for k in acc}, cntU=torch.int32, cntI=torch.int64))
        v = views(buf, lay, {p + s: torch.float32 for p in "mv" for s in keys.values() if p + s in lay})
        if self.opt != "sgd":
            self.mom = {k: (v["m" + s], v.get("v" + s)) for k, s in keys.items()}
        torch.cuda.synchronize()

    def clean(self):
        torch.cuda.synchronize()
        return all(int(torch.count_nonzero(v)) == 0 for v in self.acc.values())


class NfmGpu(_Gpu):
    def __init__(self, U, I, P, Q, bias, N, Rs, planes, L, bn, act, opt, lr, reg, td=0, max_rows=None, dropout=0.0):
        from daisyrec_b200 import _lib, ops
        self.ops, self.L, self.bn, self.act, self.opt, self.lr, self.reg, self.td = ops, L, bn, act, opt, lr, reg, td
        self.dropout = dropout
        self.P, self.Q, self.bias, self.N = (device_tensor(a).float().clone().contiguous() for a in (P, Q, bias, N))
        self.Rs = device_tensor(Rs).float().clone().contiguous() if bn else torch.zeros(0, device="cuda")
        self.t = dict(P=self.P, Q=self.Q, bias=self.bias, N=self.N, Rs=self.Rs)
        self._model("nfm", U, I, self.P.shape[1])
        self.planes = tuple(device_tensor(p).to(torch.int32).contiguous() for p in planes)
        self.max_rows = max_rows or 2 * max(2, self.planes[0].numel())
        self.hp = ops.hyper(lr, reg[0], reg[1], opt)
        self.ws = ops.NfmWorkspace(U, I, self.F, L, bn, opt, self.max_rows, "cuda")
        lay, total = nfm_ws_layout(U, I, self.F, L, bn, opt, self.max_rows)
        assert total == _lib.lib().drb_nfm_workspace_bytes(U, I, self.F, L, 1 if bn else 0, _lib.OPT_KIND[opt], self.max_rows)
        self._workspace(self.ws.buf, lay, dict(P="P", Q="Q", bias="B", N="N"))

    def run(self, lo, n, batch, k, adam_step0=0, apply=True, first_step=0, keep=None):
        bu, bi, bj = (p[lo:lo + n] for p in self.planes)
        kw = {} if keep is None else dict(dropout=self.dropout, keep=keep.cuda().contiguous())
        out = self.ops.nfm_bpr_train_steps(self.P, self.Q, self.bias, self.N, self.Rs if self.bn else None, self.ws,
                                           self.act, bu, bi, bj, batch, first_step, k, self.hp, adam_step0=adam_step0,
                                           apply=apply, tower_dtype=self.td, **kw)
        torch.cuda.synchronize()
        return out.cpu().numpy()


class NfmPhiloxGpu(NfmGpu):
    """NFM steps with dropout_engine 'philox': the masks are drawn on the device, step s keyed by (seed, adam_step0 + s); the
    reference takes the same masks as bytes from ops.nfm_philox_masks (run ignores them)"""
    seed = 0

    def run(self, lo, n, batch, k, adam_step0=0, apply=True, first_step=0, keep=None):
        bu, bi, bj = (p[lo:lo + n] for p in self.planes)
        out = self.ops.nfm_bpr_train_steps_philox(self.P, self.Q, self.bias, self.N, self.Rs if self.bn else None, self.ws,
                                                  self.act, bu, bi, bj, batch, first_step, k, self.hp, adam_step0=adam_step0,
                                                  apply=apply, tower_dtype=self.td, dropout=self.dropout, seed=self.seed)
        torch.cuda.synchronize()
        return out.cpu().numpy()


class FmGpu(_Gpu):
    def __init__(self, U, I, P, Q, bias, planes, loss, opt, lr, reg):
        from daisyrec_b200 import _lib, ops
        self.ops, self.loss, self.opt, self.lr, self.reg = ops, loss, opt, lr, reg
        self.P, self.Q, self.bias = (device_tensor(a).float().clone().contiguous() for a in (P, Q, bias))
        self.t = dict(P=self.P, Q=self.Q, bias=self.bias)
        self._model("fm", U, I, self.P.shape[1])
        self.planes = tuple(device_tensor(p).to(torch.int32).contiguous() for p in planes)
        self.hp = ops.hyper(lr, reg[0], reg[1], opt, loss=loss)
        self.ws = ops.FMWorkspace(U, I, self.F, opt, "cuda")
        lay, total = fm_ws_layout(U, I, self.F, opt)
        assert total == _lib.lib().drb_fm_workspace_bytes(U, I, self.F, _lib.OPT_KIND[opt])
        self._workspace(self.ws.buf, lay, dict(P="P", Q="Q", bias="B"))

    def run(self, lo, n, batch, k, adam_step0=0, apply=True, first_step=0):
        bu, bi, bj = (p[lo:lo + n] for p in self.planes)
        out = self.ops.fm_train_steps(self.P, self.Q, self.bias, self.ws, bu, bi, bj, batch, first_step, k, self.hp,
                                      adam_step0=adam_step0, apply=apply)
        torch.cuda.synchronize()
        return out.cpu().numpy()


class StandIn(_Model, fp64_step.StandIn):
    """CPU stand-in of the device: the reference in float32 (optionally with a defect)"""

    def __init__(self, model, U, I, tabs, planes, opt, lr, reg, L=0, bn=0, act=0, td=0, loss="BPR", dropout=0.0, defects=()):
        super().__init__(dict(tabs, Rs=tabs.get("Rs", np.zeros(0, np.float32))), planes, opt, lr, reg, defects)
        self.L, self.bn, self.act, self.td, self.loss, self.dropout = L, bn, act, td, loss, dropout
        self._model(model, U, I, self.t["P"].shape[1])
        self.gscale = None

    def stand_in_ref(self, idx, keep=None):
        if "drop_triple" in self.defects:
            idx = tuple(x[1:] for x in idx)
        if "dup_triple" in self.defects:
            idx = tuple(torch.cat([x, x[:1]]) for x in idx)
        r = self.reference(self.snapshot(), idx, self.kappa, torch.float32, self.defects, keep)
        if self.gscale is not None:                     # a defect: one section's gradient off by a relative factor
            key, sl, f = self.gscale
            r["g"][key][sl] *= f
        if self.bn and r["Rs"] is not None:
            self.t["Rs"] = r["Rs"].to(torch.float32)
        return r


# ---------------------------------------------------------------- problems
def nfm_net(F, L, bn, gen, scale=0.1, device="cuda"):
    """a network block like the bench's: N(0, scale), BatchNorm weights 1; running statistics (0, 1)"""
    lay, nN = nfm_layout(F, L, bn)
    N = torch.randn(nN, generator=gen, device=device) * scale
    for k, (a, b) in lay.items():
        if k.endswith(".g"):
            N[a:b] = 1.0
    Rs = torch.zeros((1 + L) * 2 * F if bn else 0, device=device)
    for k in range(1 + L if bn else 0):
        Rs[k * 2 * F + F:(k + 1) * 2 * F] = 1.0
    return N.contiguous(), Rs


def keep_bytes(gen, steps, L, B, F, p, device="cuda"):
    """host-drawn dropout masks as the device takes them: [step][call][site][B][F] uint8"""
    return (torch.rand(steps * 2 * (1 + L) * B * F, generator=gen, device=device) >= p).to(torch.uint8)


def uniform_planes(gen, U, I, n, device="cuda"):
    return tuple(torch.randint(0, m, (n,), generator=gen, device=device, dtype=torch.int32) for m in (U, I, I))


def ml20m():
    from daisyrec_b200.utils.synthetic import SHAPES
    return SHAPES["ml-20m"][:2]


@pytest.fixture(scope="module")
def gpu():
    from daisyrec_b200 import ops
    ops.require_cuda()
    return ops


# ---------------------------------------------------------------- GPU: NFM
def _nfm_bench(opt, td, dropout=0.0, seed=11, nsteps=3, lr=None, cls=NfmGpu):
    from daisyrec_b200.utils.synthetic import init_tables
    U, I = ml20m()
    F, L, B = 64, 1, 1 << 18
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    P, Q = init_tables(U, I, F, seed + 4, "cuda")
    P.mul_(10.0); Q.mul_(10.0)
    bias = torch.zeros(U + I + 1, device="cuda")
    N, Rs = nfm_net(F, L, True, g)
    planes = uniform_planes(g, U, I, nsteps * B)
    lr0, reg = (0.001, (0.0, 0.001)) if opt == "adam" else (0.05, (1e-3, 1e-3))
    st = cls(U, I, P, Q, bias, N, Rs, planes, L, True, 0, opt, lr or lr0, reg, td, max_rows=2 * B, dropout=dropout)
    return st, B, g


@pytest.mark.gpu
@pytest.mark.parametrize("td", [0, 1])
@pytest.mark.parametrize("opt", ["adam", "sgd"])
def test_nfm_bench_shape(gpu, opt, td):
    """f_nfm: ml-20m U / I, F = 64, L = 1, BatchNorm, relu, B = 2^18, tables x10; three steps from zero moments"""
    st, B, g = _nfm_bench(opt, td)
    recs = [checked_step(st, s * B, B, B, f"nfm {opt} td={td} step {s}", adam_step0=s, ref_device="cuda") for s in range(3)]
    report(f"nfm bench {opt} td={td}", recs)


@pytest.mark.gpu
@pytest.mark.parametrize("td", [0, 1])
def test_nfm_default_dropout(gpu, td):
    """p = 0.5 at the bench shape: three teacher-forced single-step launches with host-drawn masks, then one 3-step launch
    with the same masks from the same start, whose per-step losses meet the singles' float64 losses.  The end states are not
    compared: at this shape the BatchNorm gain (inv_std ~ 100 on the products) turns a relu gate that two atomics orders
    round to opposite sides of 0 into an O(lr g) difference one step later"""
    st, B, g = _nfm_bench("sgd", td, dropout=0.5, seed=21, lr=0.002)
    start = st.snapshot()
    keeps = [keep_bytes(g, 1, 1, B, 64, 0.5) for _ in range(3)]
    out = [checked_step(st, s * B, B, B, f"dropout td={td} step {s}", ref_device="cuda", keep=keeps[s], with_res=True)
           for s in range(3)]
    recs = [r for r, _ in out]
    multi = NfmGpu(st.U, st.I, start["P"], start["Q"], start["bias"], start["N"], start["Rs"], st.planes, 1, True, 0, "sgd",
                   st.lr, st.reg, td, max_rows=2 * B, dropout=0.5)
    l3 = multi.run(0, 3 * B, B, 3, keep=torch.cat(keeps))
    for s, (_, res) in enumerate(out):
        assert abs(float(l3[s]) - res["loss"]) <= kappa_of("nfm", td) * U_RND * res["lossN"] + res["lossP"], (s, l3[s], res["loss"])
    report(f"nfm dropout td={td}", recs)


@pytest.mark.gpu
@pytest.mark.parametrize("td", [0, 1])
def test_nfm_philox_dropout(gpu, td):
    """p = 0.5 at the bench shape with dropout_engine 'philox': three teacher-forced steps at global steps 4, 5, 6, each
    against nfm_ref with the keep factors of ops.nfm_philox_masks at that step (the kernels' own nfm_keep_factor)"""
    ops = gpu
    st, B, g = _nfm_bench("sgd", td, dropout=0.5, seed=25, lr=0.002, cls=NfmPhiloxGpu)
    st.seed = 0x5EED + td
    recs = [checked_step(st, s * B, B, B, f"philox td={td} step {4 + s}", adam_step0=4 + s, ref_device="cuda",
                         keep=ops.nfm_philox_masks(st.seed, 4 + s, B, st.F, st.L, 0.5, "cuda")) for s in range(3)]
    report(f"nfm philox dropout td={td}", recs)


# (F, L, act, bn, B): every F in NFM_F, L in NFM_L, activation, BatchNorm on and off and B in NFM_B at least once.  BatchNorm
# runs with L <= 1 only, and no case runs more than 3 layers: N_e is an absolute chain, and behind two Linear + BatchNorm
# layers, or eight Linear layers, it loses the power to see a 1e-3 gradient error.  test_harness_power_in_every_gpu_configuration
# asserts that power for every (bn, L, act) a GPU case runs.
NFM_F, NFM_L, NFM_B = (1, 6, 30, 64, 100, 200, 256), (0, 1, 3), (2, 3, 63, 4099)
NFM_GEOMETRY = [(1, 1, "relu", 1, 63), (6, 3, "sigmoid", 0, 4099), (6, 1, "tanh", 1, 3), (30, 3, "relu", 0, 63),
                (64, 0, "relu", 1, 3), (100, 1, "tanh", 0, 4099), (200, 3, "relu", 0, 2), (200, 1, "relu", 1, 63),
                (256, 1, "sigmoid", 1, 4099), (256, 3, "relu", 0, 63), (30, 1, "relu", 1, 2), (6, 0, "tanh", 0, 3)]
# (bn, L, act) of the other GPU cases: the bench shape, launches and crafted rows, saturation, scores, B = 1
NFM_OTHER_CONFIGS = [(1, 1, "relu"), (0, 1, "sigmoid"), (0, 1, "tanh"), (1, 1, "sigmoid"), (0, 1, "relu")]


@pytest.mark.gpu
@pytest.mark.parametrize("td", [0, 1])
@pytest.mark.parametrize("case", NFM_GEOMETRY, ids=lambda c: "F{}-L{}-{}-bn{}-B{}".format(*c))
def test_nfm_geometry(gpu, case, td):
    F, L, act, bn, B = case
    U, I = 700, 500
    g = torch.Generator(device="cuda"); g.manual_seed(F * 100 + L * 10 + bn + td)
    P = torch.randn(U, F, generator=g, device="cuda") * 0.5
    Q = torch.randn(I, F, generator=g, device="cuda") * 0.5
    bias = torch.randn(U + I + 1, generator=g, device="cuda") * 0.1
    N, Rs = nfm_net(F, L, bn, g, scale=1.0 / math.sqrt(F))
    planes = uniform_planes(g, U, I, 3 * B)
    a = ACTS.index(act)
    sgd = NfmGpu(U, I, P, Q, bias, N, Rs, planes, L, bn, a, "sgd", 0.05, (1e-3, 1e-3), td)
    recs = [checked_step(sgd, 0, B, B, f"{case} td={td} sgd", ref_device="cuda")]
    adam = NfmGpu(U, I, P, Q, bias, N, Rs, planes, L, bn, a, "adam", 0.001, (1e-3, 1e-3), td)
    recs += [checked_step(adam, s * B, B, B, f"{case} td={td} adam {s}", adam_step0=s, ref_device="cuda") for s in range(2)]
    report(f"nfm geometry {case} td={td}", recs)


@pytest.mark.gpu
@pytest.mark.parametrize("td", [0, 1])
def test_nfm_launches(gpu, td):
    """a 3-step launch without masks (first_step 1, ragged last batch) against three single launches, a loss-only call,
    crafted rows (repeated users, i == j, one item in every triple), saturated activations and BPR coefficients near 0 / -1"""
    U, I, F, L, B = 900, 600, 32, 1, 1500
    g = torch.Generator(device="cuda"); g.manual_seed(41 + td)
    P, Q = torch.randn(U, F, generator=g, device="cuda") * 0.5, torch.randn(I, F, generator=g, device="cuda") * 0.5
    bias = torch.randn(U + I + 1, generator=g, device="cuda") * 0.1
    N, Rs = nfm_net(F, L, True, g, scale=0.2)
    T = 4 * B - 700
    planes = uniform_planes(g, U, I, T)
    multi = NfmGpu(U, I, P, Q, bias, N, Rs, planes, L, True, 0, "sgd", 0.05, (1e-3, 1e-3), td)
    single = NfmGpu(U, I, P, Q, bias, N, Rs, planes, L, True, 0, "sgd", 0.05, (1e-3, 1e-3), td)
    # bf16: a rounding-midpoint flip between the two runs propagates through the next steps, so only the losses compare
    recs = launch_vs_singles(multi, single, T, B, 3, first_step=1, states=td == 0)
    recs.append(checked_step(single, 0, B, B, "loss only", apply=False, ref_device="cuda"))
    # crafted rows: half the batch on one (user, item, item) triple, i == j elsewhere, item 5 in every triple
    bu, bi, bj = (p.clone() for p in planes)
    bu[:B // 2], bi[:B // 2], bj[:B // 2] = 7, 5, 5
    bi[B // 2:B] = 5
    bj[B // 2:B - 100] = bi[B // 2:B - 100]
    crafted = NfmGpu(U, I, P, Q, bias, N, Rs, (bu, bi, bj), L, True, 0, "adam", 0.001, (1e-3, 1e-3), td)
    recs.append(checked_step(crafted, 0, B, B, "repeated users, i == j, one item", ref_device="cuda"))
    # saturation: large tables, no BatchNorm: sigmoid / tanh saturate and the BPR coefficients reach ~0 and ~-1
    for a in (1, 2):
        N2, _ = nfm_net(F, L, False, g, scale=1.0)
        sat = NfmGpu(U, I, P * 4, Q * 4, bias, N2 * 3, torch.zeros(0), planes, L, False, a, "sgd", 0.05, (1e-3, 1e-3), td)
        r, res = checked_step(sat, 0, B, B, f"saturated {ACTS[a]}", ref_device="cuda", with_res=True)
        recs.append(r)
    report(f"nfm launches td={td}", recs)


@pytest.mark.gpu
@pytest.mark.parametrize("td", [0, 1])
def test_nfm_scores(gpu, td):
    """drb_nfm_scores from a trained state (running statistics moved), n not a multiple of max_rows"""
    from daisyrec_b200 import ops
    U, I, F, L, B = 500, 400, 48, 1, 1000
    g = torch.Generator(device="cuda"); g.manual_seed(61 + td)
    P, Q = torch.randn(U, F, generator=g, device="cuda") * 0.5, torch.randn(I, F, generator=g, device="cuda") * 0.5
    bias = torch.randn(U + I + 1, generator=g, device="cuda") * 0.1
    N, Rs = nfm_net(F, L, True, g, scale=0.2)
    st = NfmGpu(U, I, P, Q, bias, N, Rs, uniform_planes(g, U, I, 3 * B), L, True, 1, "adam", 0.01, (0.0, 0.0), td)
    st.run(0, 3 * B, B, 3)
    assert not torch.equal(st.Rs, Rs)
    n = 10007
    u = torch.randint(0, U, (n,), generator=g, device="cuda", dtype=torch.int32)
    i = torch.randint(0, I, (n,), generator=g, device="cuda", dtype=torch.int32)
    want, wN, wP = nfm_scores_ref(st.P, st.Q, st.bias, st.N, st.Rs, U, I, L, True, 1, u.long(), i.long(), td)
    worst = 0.0
    for mr in (2, 3, 4099):
        ws = ops.NfmWorkspace(U, I, F, L, True, "sgd", mr, "cuda")
        got = ops.nfm_scores(st.P, st.Q, st.bias, st.N, st.Rs, ws, 1, u, i, tower_dtype=td).to(F64)
        err = (got - want).abs()
        r = float((err / (kappa_of("nfm", td) * U_RND * wN + wP + 2 * U_RND * want.abs())).max())
        worst = max(worst, r)
        assert r <= 1, (mr, r)
    print(f"nfm scores td={td}: worst error/bound {worst:.3g}")


@pytest.mark.gpu
def test_nfm_batchnorm_single_row(gpu):
    """with batch_norm a half of one row is refused before the first launch (torch's ValueError), apply on or off, and the
    state is bit-identical; fit on k * batch + 1 rows raises; without BatchNorm B = 1 trains and meets the fp64 bound"""
    import logging
    from daisyrec_b200.model import NFM
    from daisyrec_b200.utils.dataset import BasicDataset, get_dataloader
    U, I, F, L = 50, 40, 16, 1
    g = torch.Generator(device="cuda"); g.manual_seed(3)
    P, Q = torch.randn(U, F, generator=g, device="cuda"), torch.randn(I, F, generator=g, device="cuda")
    bias = torch.zeros(U + I + 1, device="cuda")
    N, Rs = nfm_net(F, L, True, g)
    planes = uniform_planes(g, U, I, 9)
    st = NfmGpu(U, I, P, Q, bias, N, Rs, planes, L, True, 0, "adam", 0.01, (1e-3, 1e-3))
    before = st.snapshot()
    for apply in (True, False):
        with pytest.raises(ValueError, match="Expected more than 1 value per channel"):
            st.run(8, 1, 1, 1, apply=apply)
    with pytest.raises(ValueError, match="Expected more than 1 value per channel"):
        st.run(0, 9, 4, 3)                                               # steps of 4, 4 and 1 rows: nothing runs
    after = st.snapshot()
    assert all(torch.equal(before[k], after[k]) for k in before)
    assert st.clean()
    cfg = dict(gpu="", logger=logging.getLogger("t"), epochs=1, lr=0.01, reg_1=0.0, reg_2=0.0, user_num=U, item_num=I, factors=F,
               num_layers=L, batch_norm=True, act_function="relu", dropout=0.0, loss_type="BPR", optimizer="sgd",
               init_method="default", early_stop=False, topk=10, progress=False)
    rows = np.stack([np.arange(9) % U, np.arange(9) % I, (np.arange(9) + 3) % I], 1).astype(np.int32)
    m = NFM(cfg)
    with pytest.raises(ValueError, match="Expected more than 1 value per channel"):
        m.fit(get_dataloader(BasicDataset(rows), batch_size=4, shuffle=False))
    with pytest.raises(ValueError, match="Expected more than 1 value per channel"):
        m.calc_loss([torch.from_numpy(rows[:1, k]) for k in range(3)])
    m2 = NFM(dict(cfg, batch_norm=False))
    m2.fit(get_dataloader(BasicDataset(rows), batch_size=4, shuffle=False))
    N0, _ = nfm_net(F, L, False, g)
    one = NfmGpu(U, I, P, Q, bias, N0, torch.zeros(0), planes, L, False, 0, "sgd", 0.05, (1e-3, 1e-3))
    recs = [checked_step(one, 0, 1, 1, "B = 1 without BatchNorm", ref_device="cuda")]
    report("nfm B = 1", recs)


# ---------------------------------------------------------------- GPU: FM
def _fm_problem(seed, U, I, F, n, scale=0.1, device="cuda"):
    g = torch.Generator(device=device); g.manual_seed(seed)
    P = torch.randn(U, F, generator=g, device=device) * scale
    Q = torch.randn(I, F, generator=g, device=device) * scale
    bias = torch.randn(U + I + 1, generator=g, device=device) * 0.1
    return P, Q, bias, uniform_planes(g, U, I, n, device), g


@pytest.mark.gpu
@pytest.mark.parametrize("opt", ["sgd", "adam"])
def test_fm_bench_shape(gpu, opt):
    """f_fm: ml-20m, F = 64, B = 2^20; three steps"""
    from daisyrec_b200.utils.synthetic import init_tables
    U, I = ml20m()
    B = 1 << 20
    g = torch.Generator(device="cuda"); g.manual_seed(5)
    P, Q = init_tables(U, I, 64, 7, "cuda")
    bias = torch.zeros(U + I + 1, device="cuda")
    planes = uniform_planes(g, U, I, 3 * B)
    lr = 0.01 if opt == "sgd" else 0.001
    st = FmGpu(U, I, P, Q, bias, planes, "BPR", opt, lr, (1e-3, 1e-3))
    recs = [checked_step(st, s * B, B, B, f"fm bench {opt} step {s}", adam_step0=s, ref_device="cuda") for s in range(3)]
    report(f"fm bench {opt}", recs)


def fm_planes(loss, planes, g, I):
    """CL: 0 / 1 labels; SL: small integer labels; the others: negative items"""
    bu, bi, bj = planes
    if loss == "CL":
        bj = torch.randint(0, 2, bj.shape, generator=g, device=bj.device, dtype=torch.int32)
    elif loss == "SL":
        bj = torch.randint(0, 5, bj.shape, generator=g, device=bj.device, dtype=torch.int32)
    return bu, bi, bj


FM_CASES = [(loss, opt, (32, 64, 100)[(i * 4 + j) % 3]) for i, loss in enumerate(FM_LOSSES) for j, opt in enumerate(OPTS)]


@pytest.mark.gpu
@pytest.mark.parametrize("loss,opt,F", FM_CASES)
def test_fm_loss_optimiser(gpu, loss, opt, F):
    """every loss x every optimiser at U = 20 000, I = 5 000, B = 65 573: a full step and a ragged one"""
    U, I, B = 20000, 5000, 65573
    n = 2 * B - 20000
    P, Q, bias, planes, g = _fm_problem(F + len(loss) + OPTS.index(opt), U, I, F, n, scale=0.3)
    planes = fm_planes(loss, planes, g, I)
    lr = {"sgd": 0.05, "adam": 0.001, "adagrad": 0.01, "rmsprop": 0.001}[opt]
    st = FmGpu(U, I, P, Q, bias, planes, loss, opt, lr, (1e-3, 2e-3))
    recs = [checked_step(st, 0, B, B, f"{loss} {opt} F={F} step 0", ref_device="cuda"),
            checked_step(st, B, n - B, B, f"{loss} {opt} F={F} ragged step 1", adam_step0=1, ref_device="cuda")]
    report(f"fm {loss} {opt}", recs)


def hl_margin_case(device):
    """dyadic rows with pos - neg == 1 exactly on the first 8 triples: p = e0, q_i = 1.5 e0, q_j = 0.5 e0, zero biases"""
    U, I, F = 16, 24, 8
    P, Q = torch.zeros(U, F, device=device), torch.zeros(I, F, device=device)
    P[:, 0] = 1.0
    Q[:8, 0], Q[8:16, 0] = 1.5, 0.5
    Q[16:, 1] = 0.25
    bias = torch.zeros(U + I + 1, device=device)
    bu = torch.arange(8, dtype=torch.int32, device=device)
    bi, bj = bu.clone(), bu + 8
    return U, I, P, Q, bias, (bu, bi, bj)


def hl_margin_check(st):
    """one SGD step at lr 0.25: the exact-margin triples take the gradient -1 / +1"""
    U = st.U
    st.run(0, 8, 8, 1)
    s = st.snapshot()
    P, Q, b = s["P"].cpu(), s["Q"].cpu(), s["bias"].cpu()
    want_p = torch.zeros_like(P); want_p[:, 0] = 1.0; want_p[:8, 0] = 1.25      # p - lr (-q_i + q_j)
    ok = torch.equal(P, want_p)
    ok &= bool((Q[:8, 0] == 1.75).all() and (Q[8:16, 0] == 0.25).all())          # q_i + lr p, q_j - lr p
    ok &= bool((b[U:U + 8] == 0.25).all() and (b[U + 8:U + 16] == -0.25).all() and (b[:U] == 0).all())
    return ok


@pytest.mark.gpu
def test_fm_hl_exact_margin(gpu):
    U, I, P, Q, bias, planes = hl_margin_case("cuda")
    st = FmGpu(U, I, P, Q, bias, planes, "HL", "sgd", 0.25, (0.0, 0.0))
    assert hl_margin_check(st)


@pytest.mark.gpu
@pytest.mark.parametrize("loss", ["CL", "SL"])
def test_fm_pointwise_labels(gpu, loss):
    """labels 0 / 1 (CL) and small integers (SL): item 0's row and i_bias receive nothing from the label plane"""
    U, I, F, B = 3000, 800, 64, 20000
    P, Q, bias, planes, g = _fm_problem(17 + len(loss), U, I, F, B, scale=0.3)
    bu, bi, bj = fm_planes(loss, planes, g, I)
    bi = torch.where(bi < 5, bi + 5, bi)                                 # items 0..4 never appear as items
    st = FmGpu(U, I, P, Q, bias, (bu, bi, bj), loss, "sgd", 0.05, (1e-3, 1e-3))
    pre = st.snapshot()
    r = checked_step(st, 0, B, B, f"{loss} labels", ref_device="cuda")
    post = st.snapshot()
    assert torch.equal(pre["Q"][:5], post["Q"][:5]) and torch.equal(pre["bias"][U:U + 5], post["bias"][U:U + 5])
    report(f"fm labels {loss}", [r])


@pytest.mark.gpu
@pytest.mark.parametrize("loss", FM_LOSSES)
def test_fm_launches(gpu, loss):
    """a 3-step launch (ragged last batch) against three single launches, then a loss-only call"""
    U, I, F, B = 4000, 1500, 64, 7000
    T = 3 * B - 1234
    P, Q, bias, planes, g = _fm_problem(29 + len(loss), U, I, F, T, scale=0.3)
    planes = fm_planes(loss, planes, g, I)
    multi = FmGpu(U, I, P, Q, bias, planes, loss, "adagrad", 0.01, (1e-3, 1e-3))
    single = FmGpu(U, I, P, Q, bias, planes, loss, "adagrad", 0.01, (1e-3, 1e-3))
    recs = launch_vs_singles(multi, single, T, B, 3, states=False)
    for k, a in multi.snapshot().items():
        b = single.snapshot()[k]
        assert float(((a - b).abs() / b.abs().clamp(min=1.0)).max()) <= 1e-5, k
    recs.append(checked_step(single, 0, B, B, f"{loss} loss only", adam_step0=3, apply=False, ref_device="cuda"))
    report(f"fm launches {loss}", recs)


# ---------------------------------------------------------------- CPU checks
def test_geometry_table_covers_every_value():
    cols = list(zip(*NFM_GEOMETRY))
    assert set(cols[0]) == set(NFM_F) and set(cols[1]) == set(NFM_L) and set(cols[2]) == set(ACTS)
    assert set(cols[3]) == {0, 1} and set(cols[4]) == set(NFM_B)
    assert {30, 100, 200} <= set(cols[0]) and {6, 30} <= {f for f in cols[0] if f % 4} and {200, 256} <= set(cols[0])
    assert all(L <= 1 for F, L, act, bn, B in NFM_GEOMETRY if bn)
    # every F that selects a GEMM path (scalar bf16 staging: 6, 30; the NT = 256 tile: 200, 256) runs with a hidden layer
    assert {6, 30, 200, 256} <= {F for F, L, act, bn, B in NFM_GEOMETRY if L >= 1}
    assert {loss for loss, _, _ in FM_CASES} == set(FM_LOSSES) and {o for _, o, _ in FM_CASES} == set(OPTS)
    assert {F for _, _, F in FM_CASES} == {32, 64, 100}


def test_workspace_mirrors_match_library():
    from daisyrec_b200 import _lib
    lib = _lib.lib()
    for U, I, F, L, bn, opt, mr in [(1, 1, 1, 0, 0, "sgd", 2), (7, 5, 6, 3, 1, "adam", 9), (40, 60, 30, 8, 1, "adam", 258),
                                    (138493, 26744, 64, 1, 1, "adam", 1 << 19), (300, 200, 200, 3, 0, "sgd", 8198),
                                    (11, 13, 256, 8, 1, "sgd", 126), (5, 3, 100, 1, 0, "adam", 3)]:
        assert nfm_ws_layout(U, I, F, L, bn, opt, mr)[1] == lib.drb_nfm_workspace_bytes(U, I, F, L, bn, _lib.OPT_KIND[opt], mr)
        assert nfm_layout(F, L, bn)[1] == lib.drb_nfm_param_count(F, L, bn)
    for U, I, F in [(1, 1, 1), (40, 60, 8), (20000, 5000, 100), (138493, 26744, 64)]:
        for opt in OPTS:
            assert fm_ws_layout(U, I, F, opt)[1] == lib.drb_fm_workspace_bytes(U, I, F, _lib.OPT_KIND[opt])


def _fixture_trajectory(name, c, orc=None):
    from conftest import golden
    g = golden(name)
    h = g[f"c{c}_hyper"]
    L, bn, act, lr, r1, r2, opt = int(h[0]), int(h[1]), int(h[2]), float(h[3]), float(h[4]), float(h[5]), int(h[6])
    drop, seed = (float(h[7]), int(h[8])) if name == "nfm_dropout" else (0.0, 0)
    return g, L, bn, act, lr, (r1, r2), "sgd" if opt == 0 else "adam", drop, seed


@pytest.mark.parametrize("name,c", [("nfm", c) for c in range(5)] + [("nfm_dropout", c) for c in range(5)])
def test_nfm_reference_matches_fixture(orc, name, c):
    """the unrounded reference reproduces daisyRec's three steps (losses, parameters, running statistics) from each of the
    fixture's states; under Adam the moments are the reference's own, from zero"""
    g, L, bn, act, lr, reg, opt, drop, seed = _fixture_trajectory(name, c)
    Ps, Qs, Bs, Ns, Rs = (torch.from_numpy(g[f"c{c}_{k}"]) for k in ("P", "Q", "bias", "N", "R"))
    bs, losses = g[f"c{c}_batches"], g[f"c{c}_loss"]
    U, F = Ps.shape[1:]
    I = Qs.shape[1]
    if drop:
        torch.manual_seed(seed + 100)
    mom = None
    for s in range(bs.shape[0]):
        idx = [torch.from_numpy(bs[s][k].astype(np.int64)) for k in range(3)]
        keep = None
        if drop:
            kp, kn = orc.nfm_dropout_keep(bs.shape[2], F, L, drop)
            keep = torch.cat([torch.from_numpy(kp), torch.from_numpy(kn)], 1).to(F64)
        res = nfm_ref(Ps[s], Qs[s], Bs[s], Ns[s], Rs[s], U, I, L, bn, act, *idx, reg, 0, keep)
        assert abs(res["loss"] - losses[s]) <= 3e-6 * abs(losses[s]), (s, res["loss"], losses[s])
        if bn:
            np.testing.assert_allclose(res["Rs"].numpy(), Rs[s + 1].numpy(), rtol=2e-5, atol=2e-6)
        for key, T in (("P", Ps), ("Q", Qs), ("bias", Bs), ("N", Ns)):
            th, gq, want = T[s].to(F64), res["g"][key], T[s + 1].to(F64)
            if mom is None or key not in mom:
                mom = mom or {}
                mom[key] = (torch.zeros_like(th), torch.zeros_like(th)) if opt == "adam" else None
            got, st_ = opt_apply(th, gq, mom[key], lr, opt, s + 1)
            mom[key] = st_
            err = (got - want).abs()
            # Adam: slots whose gradient is fp32 cancellation noise in the reference's run take +-lr steps of either sign
            noise = (gq.abs() <= 1e-5 * float(gq.abs().max())) if opt == "adam" else torch.zeros_like(err, dtype=torch.bool)
            tol = 2e-6 * max(1.0, float(want.abs().max()))
            assert float(err[~noise].max()) <= tol, (key, s, float(err[~noise].max()))


@pytest.mark.parametrize("c", range(5))
def test_fm_reference_matches_fixture(c):
    from conftest import golden
    g = golden("fm")
    lr, r1, r2 = (float(x) for x in g[f"c{c}_hyper"])
    opt, loss = str(g[f"c{c}_opt"]), str(g[f"c{c}_losskind"])
    Ps, Qs, Bs = (torch.from_numpy(g[f"c{c}_{k}"]) for k in ("P", "Q", "bias"))
    bs, losses = g[f"c{c}_batches"], g[f"c{c}_loss"]
    U, I = Ps.shape[1], Qs.shape[1]
    mom = {}
    for s in range(bs.shape[0]):
        idx = [torch.from_numpy(bs[s][k].astype(np.int64)) for k in range(3)]
        res = fm_ref(Ps[s], Qs[s], Bs[s], U, I, *idx, loss, (r1, r2))
        assert abs(res["loss"] - losses[s]) <= 3e-6 * abs(losses[s]), (s, res["loss"], losses[s])
        for key, T in (("P", Ps), ("Q", Qs), ("bias", Bs)):
            th, gq, want = T[s].to(F64), res["g"][key], T[s + 1].to(F64)
            if key not in mom:
                mom[key] = (torch.zeros_like(th), torch.zeros_like(th)) if opt == "adam" else None
            got, mom[key] = opt_apply(th, gq, mom[key], lr, opt, s + 1)
            noise = (gq.abs() <= 1e-5 * float(gq.abs().max())) if opt == "adam" else torch.zeros_like(th, dtype=torch.bool)
            err = (got - want).abs()
            assert float(err[~noise].max()) <= 2e-6 * max(1.0, float(want.abs().max())), (key, s, float(err[~noise].max()))


def _cpu_nfm(opt="sgd", td=0, L=2, bn=1, act=0, F=16, B=300, reg=(1e-3, 1e-3), dropout=0.0, defects=(), seed=5):
    rng = np.random.default_rng(seed)
    U, I = 120, 90
    lay, nN = nfm_layout(F, L, bn)
    N = (rng.standard_normal(nN) * 0.3).astype(np.float32)
    for k, (a, b) in lay.items():
        if k.endswith(".g"):
            N[a:b] = 1.0 + 0.1 * rng.standard_normal(b - a)
    Rs = np.tile(np.concatenate([np.zeros(F), np.ones(F)]), 1 + L if bn else 0).astype(np.float32)
    tabs = dict(P=(rng.standard_normal((U, F)) * 0.5).astype(np.float32), Q=(rng.standard_normal((I, F)) * 0.5).astype(np.float32),
                bias=(rng.standard_normal(U + I + 1) * 0.1).astype(np.float32), N=N, Rs=Rs)
    planes = (rng.integers(U, size=2 * B), rng.integers(I, size=2 * B), rng.integers(I, size=2 * B))
    lr = 0.05 if opt == "sgd" else 0.01
    return StandIn("nfm", U, I, tabs, planes, opt, lr, reg, L, bn, act, td, dropout=dropout, defects=defects), B


def _cpu_fm(loss="BPR", opt="sgd", F=16, B=400, reg=(1e-3, 2e-3), defects=(), seed=7):
    rng = np.random.default_rng(seed)
    U, I = 150, 100
    tabs = dict(P=(rng.standard_normal((U, F)) * 0.4).astype(np.float32), Q=(rng.standard_normal((I, F)) * 0.4).astype(np.float32),
                bias=(rng.standard_normal(U + I + 1) * 0.1).astype(np.float32))
    bj = rng.integers(I, size=2 * B) if loss not in ("CL", "SL") else rng.integers(2 if loss == "CL" else 5, size=2 * B)
    bi = rng.integers(I, size=2 * B)
    if loss in ("CL", "SL"):
        bi = np.maximum(bi, 5)
    planes = (rng.integers(U, size=2 * B), bi, bj)
    lr = {"sgd": 0.05, "adam": 0.01, "adagrad": 0.01, "rmsprop": 0.001}[opt]
    return StandIn("fm", U, I, tabs, planes, opt, lr, reg, loss=loss, defects=defects), B


@pytest.mark.parametrize("opt,td,act,bn", [("sgd", 0, 0, 1), ("adam", 0, 0, 1), ("sgd", 1, 0, 1), ("adam", 1, 1, 1),
                                           ("sgd", 0, 2, 0), ("adam", 1, 2, 0)])
def test_harness_passes_with_fp32_stand_in_nfm(opt, td, act, bn):
    st, B = _cpu_nfm(opt, td, act=act, bn=bn)
    for s in range(2):
        r = checked_step(st, s * B, B, B, f"stand-in nfm {opt} td={td} {s}", adam_step0=s)
        assert r["ok"], summary(r)


def test_harness_passes_with_fp32_stand_in_nfm_dropout():
    st, B = _cpu_nfm("sgd", 0, dropout=0.5)
    g = torch.Generator(); g.manual_seed(1)
    for s in range(2):
        r = checked_step(st, s * B, B, B, f"stand-in nfm dropout {s}", keep=keep_bytes(g, 1, st.L, B, st.F, 0.5, "cpu"))
        assert r["ok"], summary(r)


@pytest.mark.parametrize("loss,opt", [(loss, opt) for loss in FM_LOSSES for opt in OPTS])
def test_harness_passes_with_fp32_stand_in_fm(loss, opt):
    st, B = _cpu_fm(loss, opt)
    for s in range(2):
        r = checked_step(st, s * B, B, B, f"stand-in fm {loss} {opt} {s}", adam_step0=s)
        assert r["ok"], summary(r)


DEFECTS = {
    # defect: (model, optimiser, tower dtype / loss, extra)
    "drop_triple": ("nfm", "sgd", 0, {}),
    "dup_triple": ("nfm", "sgd", 0, {}),
    "bn_all_rows": ("nfm", "sgd", 0, {}),
    "biased_running_var": ("nfm", "sgd", 0, {}),
    "neg_running_first": ("nfm", "sgd", 0, {}),
    "sigmoid_from_z": ("nfm", "sgd", 0, dict(act=1)),
    "ubias_per_half": ("nfm", "adam", 0, {}),
    "unrounded_h": ("nfm", "sgd", 1, dict(bn=0, L=1)),
    "unrounded_W": ("nfm", "sgd", 1, dict(bn=0, L=1)),
    "unrounded_hprev": ("nfm", "sgd", 1, dict(bn=0, L=1)),
    "unrounded_dz": ("nfm", "sgd", 1, dict(bn=0, L=1)),
    "unrounded_dzi": ("nfm", "sgd", 1, dict(bn=0, L=1)),
    "unrounded_Wi": ("nfm", "sgd", 1, dict(bn=0, L=1)),
    "label_scatter": ("fm", "sgd", "CL", {}),
}


@pytest.mark.parametrize("defect", sorted(DEFECTS))
def test_harness_flags_defective_stand_in(defect):
    model, opt, x, kw = DEFECTS[defect]
    if model == "nfm":
        st, B = _cpu_nfm(opt, x, defects=(defect,), **kw)
    else:
        st, B = _cpu_fm(x, opt, defects=(defect,))
    r = checked_step(st, 0, B, B, defect)
    worst = max([r.get("ratio", 0.0), r["loss_ratio"], r["checks"]["rs_ratio"]])
    print(f"{defect}: ok={r['ok']} worst ratio {worst:.3g} bias_exact={r['checks'].get('bias_exact')} "
          f"stray={sum(c.get('stray', 0) for c in r['tensors'].values())}")
    assert not r["ok"], summary(r)


def test_harness_flags_hl_cut_at_equality():
    """HL's gradient cut at equality (m > 0 instead of m >= 0): the dyadic exact-margin check fails, the correct one passes"""
    U, I, P, Q, bias, planes = hl_margin_case("cpu")
    tabs = dict(P=P.numpy(), Q=Q.numpy(), bias=bias.numpy())
    good = StandIn("fm", U, I, tabs, [p.numpy() for p in planes], "sgd", 0.25, (0.0, 0.0), loss="HL")
    assert hl_margin_check(good)
    bad = StandIn("fm", U, I, tabs, [p.numpy() for p in planes], "sgd", 0.25, (0.0, 0.0), loss="HL", defects=("hl_cut",))
    assert not hl_margin_check(bad)


POWER_SECTIONS = ("P", "W0", "wp", "bn0.g")
UNROUNDED = ("unrounded_h", "unrounded_W", "unrounded_hprev", "unrounded_dz", "unrounded_dzi", "unrounded_Wi")


@pytest.mark.parametrize("td", [0, 1])
@pytest.mark.parametrize("cfg", sorted({(bn, L, act) for F, L, act, bn, B in NFM_GEOMETRY} | set(NFM_OTHER_CONFIGS)),
                         ids=lambda c: "bn{}-L{}-{}".format(*c))
def test_harness_power_in_every_gpu_configuration(cfg, td):
    """in every (BatchNorm, layers, activation) a GPU case runs: one section's gradient off by 1e-3 relative (5e-3 in bf16,
    where BN0's gamma behind sigmoid / tanh needs it), and (bf16) each GEMM operand left unrounded in layer 0, exceed the
    bound; the correct stand-in passes"""
    bn, L, act = cfg
    a = ACTS.index(act)
    st, B = _cpu_nfm("sgd", td, L=L, bn=bn, act=a)
    r = checked_step(st, 0, B, B, "correct", ladder=False)
    assert r["ok"], summary(r)
    ratios, rel = {}, 1e-3 if td == 0 else 5e-3
    for key in POWER_SECTIONS:
        if (key == "W0" and L == 0) or (key == "bn0.g" and not bn):
            continue
        st, B = _cpu_nfm("sgd", td, L=L, bn=bn, act=a)
        if key in ("P", "Q"):
            st.gscale = (key, slice(None), 1 + rel)
        else:
            lo, hi = nfm_layout(st.F, L, bn)[0][key]
            st.gscale = ("N", slice(lo, hi), 1 + rel)
        ratios[key] = checked_step(st, 0, B, B, key, ladder=False).get("ratio", 0.0)
    for d in (UNROUNDED if td == 1 and L >= 1 else ()):
        st, B = _cpu_nfm("sgd", td, L=L, bn=bn, act=a, defects=(d,))
        ratios[d] = checked_step(st, 0, B, B, d, ladder=False).get("ratio", 0.0)
    print(cfg, td, {k: round(v, 3) for k, v in ratios.items()})
    assert all(v > 1 for v in ratios.values()), ratios
