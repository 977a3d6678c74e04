"""The NeuMF + BPR step of the bf16 towers (tower_dtype 2: neumf_fused_kernel; tower_dtype 1: layer-wise wgmma GEMMs) against a
float64 reference that rounds to bf16 exactly where the kernels round, one teacher-forced step at a time (fp64_step.py: the
snapshot of the tables, the tower block W and the Adam moments, the bound and its checks).

Rounding points.  Fused: A0 = cat(UM[u], IM[item]), W1, W2 are rounded (identical fp32 inputs: bit-identical on both sides);
A1 = relu(Z1 + b1) is rounded and its ReLU gate is read from the rounded value; h = relu(Z2 + b2) stays fp32; dZ2 and dZ1 are
rounded; the weight-gradient and dA0 products take the rounded operands; bias / predict-layer / GMF gradients, loss and norms
come from the fp32 values before rounding.  Layer-wise: each GEMM rounds its two operands iff `gemm_bf16(dtype, N)` (the
dispatcher's rule, N as passed at each call site), everything else is fp32.  The fused path is the layer-wise rule with every
GEMM rounded (a ReLU gate read from bf16(a) or from a is the same gate), so one reference serves both.

N_e ("A_e") runs |A0| |W1|^T ... down to |dZ1|^T |A0|.  P_e ("Phi_e"): a rounded value that may round to its neighbour, a
ReLU gate that may go either way (delta = the whole gated value); the error of x reaches the BPR coefficient through
|dc/dx| <= 1/4.  P_e is a worst-case sum: on sums over many rows (the weight and bias gradients) it is much wider than the
KAPPA term, so an error of bf16-rounding size spread over such a sum (for example a bias gradient summed from the rounded
instead of the fp32 values) is not always caught there; errors of a lost or misplaced contribution, a wrong rounding point in
a product, or the wrong regulariser norm are (the defective stand-ins below).  Under SGD the elements with no contribution
are untouched rows, dead units and the predict bias.  The gradient accumulators and row counters are zero after every step.
"""
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)
import fp64_step  # noqa: E402
from fp64_step import (F64, GAMMA, U_RND, Flags, Stepper, _A, adam_apply, br, carve, checked_step,  # noqa: E402
                       device_tensor, launch_vs_singles, report, rnd, summary, views)

# Calibrated on one H100 80GB HBM3 (700 W power limit) over every case below: the largest KAPPA any element without a discrete
# term needed was 5.9 (layer-wise F = 4, L = 1, B = 20 000, one item-table element; 1.6 at most elsewhere), hence 12 (about 2x).
# At KAPPA = 12 at most 13 % of the rounded or gated intermediates of a step lie within their noise of a bf16 midpoint or of
# the ReLU kink (F = 128, L = 3; 0.2 - 2.8 % along the bench trajectory), hence the 26 % ceiling on that fraction.
KAPPA = 12.0
PHI_FRAC_MAX = 0.26
NAMES = ("UG", "IG", "UM", "IM", "W")
UMMA_MAX_N = 256


# ---------------------------------------------------------------- mirrors of the path selection (neumf.cu, neumf_fused.cuh)
def fused_supported(F, L, mode, dropout):
    """neumf_fused_supported"""
    return L == 2 and mode == 0 and dropout == 0.0 and F == 32


def gemm_bf16(dtype, N):
    """launch_gemm: wgmma (bf16 operands) iff dtype == 1 and N <= kUmmaMaxN, decided per call"""
    return dtype == 1 and N <= UMMA_MAX_N


def widths(F, L):
    D = F << (L - 1)
    return [2 * D >> l for l in range(L + 1)]


def tower_plan(tower_dtype, F, L, mode=0, dropout=0.0):
    """which tower GEMMs round their operands.  fwd[l]: A_l W_l^T (N = n[l+1]); wg[l]: A_l^T dZ (N = n[l+1]); ig[l]: dZ W_l
    (N = n[l]).  tower_dtype 2 outside the fused kernel's shapes runs the layer-wise bf16 path."""
    n = widths(F, L)
    fused = tower_dtype == 2 and fused_supported(F, L, mode, dropout)
    dt = 1 if tower_dtype == 2 else tower_dtype
    if fused:
        return dict(fused=True, fwd=[True] * L, wg=[True] * L, ig=[True] * L)
    return dict(fused=False, fwd=[gemm_bf16(dt, n[l + 1]) for l in range(L)], wg=[gemm_bf16(dt, n[l + 1]) for l in range(L)],
                ig=[gemm_bf16(dt, n[l]) for l in range(L)])


def layout(F, L, mode=0):
    n = widths(F, L)
    w_off, b_off, o = [], [], 0
    for l in range(L):
        w_off.append(o); o += n[l] * n[l + 1]
        b_off.append(o); o += n[l + 1]
    wp_off = o
    o += (2 if mode == 0 else 1) * F
    return dict(n=n, w_off=w_off, b_off=b_off, wp_off=wp_off, bp_off=o, nW=o + 1)


def fused_geometry(B, sms):
    tiles = -(-B // 64)
    grid = max(1, min(tiles, sms))
    return dict(tiles=tiles, grid=grid, per_cta=-(-tiles // grid), partial=B % 64 != 0)


# ---------------------------------------------------------------- the reference step
def ref_step(tabs, W, bu, bi, bj, F, L, plan, mode=0, keep=None, reg=(0.0, 0.0), dt=F64, defects=(), chunk=1 << 17):
    """One NeuMF + BPR step (gradients, not applied) of the path `plan` on fp32 tables / W.  dt = float64 is the reference;
    dt = float32 is a CPU stand-in of the device (same bf16 operands, fp32 products in torch's order).  keep: the [2B, sum n_l]
    dropout keep factors (rows: pos forward, then neg forward).  -> dict(g, N, P: lists over NAMES (float64), loss, lossN, lossP,
    cnt: per-table occurrence counts)."""
    UG, IG, UM, IM = tabs
    dev = UG.device
    lay = layout(F, L, mode)
    n, D = lay["n"], F << (L - 1)
    Wd = W.to(dt)
    B = len(bu)
    if "drop_last_triple" in defects:
        bu, bi, bj = bu[:-1], bi[:-1], bj[:-1]
    T = len(bu)
    reg1, reg2 = reg
    st = Flags(KAPPA)               # rounded or gated intermediates that may round / gate the other way, of all of them
    kus = st.k * U_RND
    use_g, hoff, npw = mode != 2, (F if mode == 0 else 0), (2 if mode == 0 else 1) * F
    koff = np.concatenate([[0], np.cumsum(n[:L])]).astype(int)

    # batch norms of the regulariser: UG_u, UM_u, IG_i, IM_i, IG_j (IM_j never enters; IG_j is weighted twice)
    rows5 = [(UG, bu), (UM, bu), (IG, bi), (IM, bi), (IG, bj)]
    s2 = [float((T_[idx].to(F64) ** 2).sum()) for T_, idx in rows5]
    l1 = [float(T_[idx].to(F64).abs().sum()) for T_, idx in rows5]
    if "imj_in_norms" in defects:
        s2[3] += float((IM[bj].to(F64) ** 2).sum())
        l1[3] += float(IM[bj].to(F64).abs().sum())
    nr = [math.sqrt(s) for s in s2]
    inv = [float(np.float32(1.0 / v)) if v > 0 else 0.0 for v in nr]

    shapes = [UG.shape, IG.shape, UM.shape, IM.shape, (lay["nW"],)]
    g = [torch.zeros(s, dtype=F64, device=dev) for s in shapes]
    N = [torch.zeros(s, dtype=F64, device=dev) for s in shapes]
    P = [torch.zeros(s, dtype=F64, device=dev) for s in shapes]
    cu = torch.bincount(bu, minlength=UG.shape[0]).to(F64)[:, None]
    ci = torch.bincount(bi, minlength=IG.shape[0]).to(F64)[:, None]
    cj = torch.bincount(bj, minlength=IG.shape[0]).to(F64)[:, None]
    if reg1 or reg2:
        def term(Tt, iv):
            T64 = Tt.to(F64)
            return reg1 * torch.sign(T64) + reg2 * T64 * iv
        for k, parts in ((0, [(cu, UG, inv[0])]), (1, [(ci, IG, inv[2]), (2 * cj, IG, inv[4])]), (2, [(cu, UM, inv[1])]),
                         (3, [(ci, IM, inv[3])])):
            for c, Tt, iv in parts:
                t = term(Tt, iv)
                g[k] += c * t
                N[k] += c * t.abs()

    loss = lossN = lossP = 0.0
    Wmat = lambda l: Wd[lay["w_off"][l]:lay["w_off"][l] + n[l] * n[l + 1]].view(n[l + 1], n[l])
    bvec = lambda l: Wd[lay["b_off"][l]:lay["b_off"][l] + n[l + 1]]
    wp = Wd[lay["wp_off"]:lay["wp_off"] + npw]
    wp_g, wp_h = (wp[:F] if use_g else None), wp[hoff:hoff + F]
    for a in range(0, T, chunk):
        b = min(T, a + chunk)
        m = b - a
        u, ip, jn = bu[a:b], bi[a:b], bj[a:b]
        uu, it = torch.cat([u, u]), torch.cat([ip, jn])
        tri = torch.arange(a, b, device=dev).repeat(2)
        kp = None if keep is None else torch.cat([keep[a:b], keep[B + a:B + b]]).to(dt)
        x0 = torch.cat([UM[uu], IM[it]], 1).to(dt)
        if kp is not None:
            x0 = x0 * kp[:, :n[0]]
        acts = [(x0, torch.zeros(x0.shape, dtype=F64, device=dev), torch.zeros(x0.shape, dtype=F64, device=dev))]
        pres = [None]
        for l in range(L):
            av, aN, aP = acts[l]
            w = Wmat(l)
            if plan["fwd"][l]:
                av, aN, aP = rnd(av, aN, aP, st)
                w = br(w)
            z = av @ w.T + bvec(l)
            zN = _A(av) @ _A(w).T + _A(bvec(l)) + aN @ _A(w).T
            zP = aP @ _A(w).T
            e = kus * zN + zP
            live = z > -e
            out = torch.relu(z)
            oN, oP = torch.where(live, zN, 0.0), torch.where(live, zP, 0.0)
            pres.append((z, e))
            if kp is not None and l + 1 < L:
                kl = kp[:, koff[l + 1]:koff[l + 1] + n[l + 1]]
                out, oN, oP = out * kl, oN * _A(kl), oP * _A(kl)
            acts.append((out, oN, oP))

        # head
        h, hN, hP = acts[L]
        ug, ig = UG[uu].to(dt), IG[it].to(dt)
        pred = h @ wp_h
        predN = _A(h) @ _A(wp_h) + hN @ _A(wp_h)
        predP = hP @ _A(wp_h)
        if use_g:
            gmf = ug * ig
            pred = pred + gmf @ wp_g
            predN = predN + _A(gmf) @ _A(wp_g)
        x = pred[:m] - pred[m:]
        xN = predN[:m] + predN[m:] + _A(pred[:m]) + _A(pred[m:])
        xP = predP[:m] + predP[m:]
        s = 1.0 / (1.0 + torch.exp(-x))
        c = -(s * (1.0 - s)) / (GAMMA + s)
        lt = -torch.log(GAMMA + s)
        loss += float(lt.to(F64).sum())
        lossN += float((xN + _A(lt)).sum())
        lossP += float(xP.sum())
        dp = torch.cat([c, -c])
        dpN = torch.cat([xN / 4 + _A(c)] * 2)
        dpP = torch.cat([xP / 4] * 2)
        gw = g[4]
        o = lay["wp_off"]
        if use_g:
            v = dp[:, None] * wp_g * ig
            g[0].index_add_(0, uu, v.to(F64)); N[0].index_add_(0, uu, _A(v) + dpN[:, None] * _A(wp_g * ig))
            t_ = dpP[:, None] * _A(wp_g * ig)
            P[0].index_add_(0, uu, t_)
            v = dp[:, None] * wp_g * ug
            g[1].index_add_(0, it, v.to(F64)); N[1].index_add_(0, it, _A(v) + dpN[:, None] * _A(wp_g * ug))
            t_ = dpP[:, None] * _A(wp_g * ug)
            P[1].index_add_(0, it, t_)
            gw[o:o + F] += (dp[:, None] * gmf).to(F64).sum(0)
            N[4][o:o + F] += (_A(dp[:, None] * gmf) + dpN[:, None] * _A(gmf)).sum(0)
            t_ = dpP[:, None] * _A(gmf)
            P[4][o:o + F] += t_.sum(0)
        gw[o + hoff:o + hoff + F] += (dp[:, None] * h).to(F64).sum(0)
        N[4][o + hoff:o + hoff + F] += (_A(dp[:, None] * h) + dpN[:, None] * _A(h) + _A(dp)[:, None] * hN).sum(0)
        t_ = dpP[:, None] * _A(h) + _A(dp)[:, None] * hP
        P[4][o + hoff:o + hoff + F] += t_.sum(0)

        # dZ_L = dp wp_h [h > 0]
        zL, eL = pres[L]
        dz = dp[:, None] * wp_h
        dzN = _A(dz) + dpN[:, None] * _A(wp_h)
        dzP = dpP[:, None] * _A(wp_h)
        cur, curN, curP = _gate(dz, dzN, dzP, zL, eL, None, st)
        for l in reversed(range(L)):
            av, aN, aP = acts[l]
            w = Wmat(l)
            # gW_l += dZ^T A_l
            ca, caN, caP = av, aN, aP
            cd, cdN, cdP = cur, curN, curP
            if plan["wg"][l]:
                ca, caN, caP = rnd(av, aN, aP, st)
                if not ("dz1_unrounded" in defects and l == 0):
                    cd, cdN, cdP = rnd(cur, curN, curP, st)
            if "drop_tile_gw1" in defects and l == 0:
                keep_rows = ((tri < 64) | (tri >= 128)).to(dt)[:, None]
                cd, cdN, cdP = cd * keep_rows, cdN * keep_rows.to(F64), cdP * keep_rows.to(F64)
            wo, bo = lay["w_off"][l], lay["b_off"][l]
            gw[wo:bo] += (cd.T @ ca).to(F64).reshape(-1)
            N[4][wo:bo] += (_A(cd).T @ _A(ca) + cdN.T @ _A(ca) + _A(cd).T @ caN).reshape(-1)
            P[4][wo:bo] += (cdP.T @ _A(ca) + _A(cd).T @ caP).reshape(-1)
            # gb_l += column sums of the fp32 dZ
            cb = br(cur) if ("gb1_rounded" in defects and l == 0) else cur
            gw[bo:bo + n[l + 1]] += cb.to(F64).sum(0)
            N[4][bo:bo + n[l + 1]] += (_A(cb) + curN).sum(0)
            P[4][bo:bo + n[l + 1]] += curP.sum(0)
            # dA_l = dZ W_l
            dd, ddN, ddP, ww = cur, curN, curP, w
            if plan["ig"][l]:
                if not ("dz1_unrounded" in defects and l == 0):
                    dd, ddN, ddP = rnd(cur, curN, curP, st)
                ww = br(w)
            dv = dd @ ww
            dN = _A(dd) @ _A(ww) + ddN @ _A(ww)
            dP = ddP @ _A(ww)
            kl = None if kp is None else kp[:, koff[l]:koff[l] + n[l]]
            if l > 0:
                z, e = pres[l]
                cur, curN, curP = _gate(dv, dN, dP, z, e, kl, st)
            else:
                cur, curN, curP = dv, dN, dP
                if kl is not None:
                    cur, curN, curP = cur * kl, curN * _A(kl), curP * _A(kl)
        if "swap_da0" in defects and a == 0:
            cur = cur.clone()
            cur[0, [0, 1]] = cur[0, [1, 0]]
        g[2].index_add_(0, uu, cur[:, :D].to(F64)); N[2].index_add_(0, uu, _A(cur[:, :D]) + curN[:, :D])
        P[2].index_add_(0, uu, curP[:, :D])
        g[3].index_add_(0, it, cur[:, D:].to(F64)); N[3].index_add_(0, it, _A(cur[:, D:]) + curN[:, D:])
        P[3].index_add_(0, it, curP[:, D:])

    # the loss as neumf_finalize_kernel assembles it
    lreg = reg1 * (l1[2] + l1[4]) + reg1 * (l1[3] + l1[4]) + reg2 * (nr[2] + nr[4]) + reg2 * (nr[3] + nr[4]) \
        + reg1 * l1[0] + reg1 * l1[1] + reg2 * nr[0] + reg2 * nr[1]
    return dict(g=g, N=N, P=P, loss=loss + lreg, lossN=lossN + abs(lreg) + abs(loss + lreg), lossP=lossP,
                cnt=(cu, ci + cj, cu, ci + cj), flagged=st.frac())


def _gate(d, dN, dP, z, e, kl, st):
    """d [z > 0] (x keep factor kl): certain where |z| > e; an uncertain gate may pass d or 0 (its whole size goes to P)"""
    kf = torch.ones((), dtype=d.dtype, device=d.device) if kl is None else kl
    ka = _A(kf)
    alive = (kf != 0) if kl is not None else torch.ones((), dtype=torch.bool, device=d.device)
    on = (z > e) & alive
    unc = (z.abs().to(F64) <= e) & alive
    out = d * (z > 0).to(d.dtype) * kf
    oN = torch.where(on, dN * ka, 0.0)
    oP = torch.where(on, dP * ka, torch.where(unc, (_A(d) + st.k * U_RND * dN + dP) * ka, 0.0))
    st.add(unc)
    return out, oN, oP


def sections(F, L, mode=0):
    """[(name, lo, hi)] of the tower block W: each layer's weight and bias, the predict weight (the predict bias has no
    gradient: it must stay bit-identical under SGD)"""
    lay = layout(F, L, mode)
    out = []
    for l in range(L):
        out += [(f"W{l + 1}", lay["w_off"][l], lay["b_off"][l]), (f"b{l + 1}", lay["b_off"][l], lay["b_off"][l] + lay["n"][l + 1])]
    return out + [("wp", lay["wp_off"], lay["bp_off"]), ("bp", lay["bp_off"], lay["nW"])]


# ---------------------------------------------------------------- steppers: the device and its CPU stand-in
def neumf_ws_parts(U, I, F, L, opt):
    """carve_neumf (neumf.cu)"""
    D, nW = F << (L - 1), layout(F, L, 0)["nW"]
    parts = [("hdrG", 256), ("hdrM", 256), ("red", 128), ("gUG", 4 * U * F), ("gIG", 4 * I * F), ("gUM", 4 * U * D),
             ("gIM", 4 * I * D), ("gW", 4 * nW), ("cntU", 4 * U), ("cntI", 8 * I)]
    if opt == "adam":
        for k, s in (("UG", U * F), ("IG", I * F), ("UM", U * D), ("IM", I * D), ("W", nW)):
            parts += [("m" + k, 4 * s), ("v" + k, 4 * s)]
    return parts


class _Neumf:
    """NeuMF on the tables UG, IG, UM, IM and the tower block W: the reference call (ref_step of the path `plan`) and the
    compared sections"""
    kappa, phi_max, ladder = KAPPA, PHI_FRAC_MAX, False     # the ladder would re-run ref_step at B = 1 M on the bench trajectory

    def reference(self, pre, idx, kappa, dt=F64, defects=(), keep=None, masks=None):
        res = ref_step([pre[k] for k in NAMES[:4]], pre["W"], *idx, self.F, self.L, self.plan, self.mode,
                       None if keep is None else keep.to(pre["W"].device), self.reg, dt, defects)
        return dict(res, **{x: dict(zip(NAMES, res[x])) for x in ("g", "N", "P")})

    def sections(self):
        return ([(k, k, 0, self.t[k].numel(), self.t[k].shape[1]) for k in NAMES[:4]]
                + [(name, "W", lo, hi, 1) for name, lo, hi in sections(self.F, self.L, self.mode)])

    def checks(self, pre, post, res, apply):
        return dict(clean=self.clean())


class GpuNeumf(_Neumf, Stepper):
    """the device step (ops.neumf_bpr_train_steps) on tables / W / planes held on `device`"""

    def __init__(self, tabs, W, planes, F, L, opt, lr, reg, max_rows, mode=0, tower_dtype=2, dropout=0.0, device="cuda"):
        from daisyrec_b200 import ops
        self.ops, self.device = ops, device
        self.F, self.L, self.opt, self.lr, self.reg, self.mode, self.td, self.dropout = F, L, opt, lr, reg, mode, tower_dtype, dropout
        self.plan = tower_plan(tower_dtype, F, L, mode, dropout)
        with torch.cuda.device(device):
            self.t = {k: device_tensor(a, device).clone().contiguous() for k, a in zip(NAMES, list(tabs) + [W])}
            self.planes = tuple(device_tensor(p, device).to(torch.int32).contiguous() for p in planes)
            U, I = self.t["UG"].shape[0], self.t["IG"].shape[0]
            self.ws = ops.NeumfWorkspace(U, I, F, L, opt, max_rows, device)
            self.hp = ops.hyper(lr, reg[0], reg[1], opt)
            torch.cuda.synchronize()
        lay, _ = carve(neumf_ws_parts(U, I, F, L, opt))
        acc = {k: torch.float32 for k in ("gUG", "gIG", "gUM", "gIM", "gW")}
        self.acc = views(self.ws.buf, lay, dict(acc, cntU=torch.int32, cntI=torch.int64))
        if opt == "adam":
            v = views(self.ws.buf, lay, {p + k: torch.float32 for k in NAMES for p in "mv"})
            self.mom = {k: (v["m" + k], v["v" + k]) for k in NAMES}

    def clean(self):
        torch.cuda.synchronize(self.device)
        return all(int(v.count_nonzero()) == 0 for v in self.acc.values())

    def run(self, lo, n, batch, k, adam_step0=0, apply=True, first_step=0, keep=None, masks=None):
        with torch.cuda.device(self.device):
            bu, bi, bj = (p[lo:lo + n] for p in self.planes)
            losses = self.ops.neumf_bpr_train_steps([self.t[k] for k in NAMES[:4]], self.t["W"], self.ws, bu, bi, bj, batch,
                                                    first_step, k, self.hp, adam_step0=adam_step0, apply=apply,
                                                    tower_dtype=self.td, dropout=self.dropout, drop_masks=masks, mode=self.mode)
            out = losses.cpu().numpy()
        torch.cuda.synchronize(self.device)
        return out


class StandIn(_Neumf, fp64_step.StandIn):
    """CPU stand-in of the device: ref_step in float32 (same bf16 operands, fp32 products in torch's order), optional
    defects"""

    def __init__(self, tabs, W, planes, F, L, opt, lr, reg, plan, mode=0, defects=()):
        super().__init__(dict(zip(NAMES, list(tabs) + [W])), planes, opt, lr, reg, defects)
        self.F, self.L, self.plan, self.mode = F, L, plan, mode


# ---------------------------------------------------------------- problems
def make_problem(rng, U, I, F, L, mode=0, tscale=0.1, wscale=0.15):
    D = F << (L - 1)
    tabs = [(rng.standard_normal(s) * tscale).astype(np.float32) for s in ((U, F), (I, F), (U, D), (I, D))]
    W = (rng.standard_normal(layout(F, L, mode)["nW"]) * wscale).astype(np.float32)
    return tabs, W


def uniform_planes(rng, U, I, n):
    return (rng.integers(U, size=n).astype(np.int32), (rng.random(n) ** 2 * I).astype(np.int32), rng.integers(I, size=n).astype(np.int32))


def host_masks(B, F, L, p, seed):
    """torch's own keep factors for one step (oracle.torch_dropout_keep) and their bit-packed device form"""
    from oracle import oracle as orc
    torch.manual_seed(seed)
    keep = orc.torch_dropout_keep(B, F, L, p)
    words, col = [], 0
    for w in widths(F, L)[:L]:
        bits = np.packbits((keep[:, col:col + w] != 0).reshape(-1), bitorder="little")
        words.append(np.pad(bits, (0, (-len(bits)) % 4)).view(np.int32))
        col += w
    return torch.from_numpy(keep), np.concatenate(words)


FUSED_CASES = ["tiles-small", "tiles-sms", "dup-user", "dup-item", "dup-mixed", "dead-units", "saturated", "reg0", "adam",
               "loss-only-65", "launch-split"]
LAYER_SHAPES = [(4, 1), (12, 2), (24, 2), (32, 2), (64, 1), (64, 3), (128, 2), (128, 3)]
LAYER_BATCHES = [1, 63, 2049, 20000]


def run_fused_case(name, make, sms, ref_device):
    """fused (tower_dtype 2) cases at F = 32, L = 2.  make(tabs, W, planes, F, L, opt, lr, reg, max_rows, ...) -> stepper."""
    F, L = 32, 2
    plan = tower_plan(2, F, L)
    assert plan["fused"]
    rng = np.random.default_rng(sum(map(ord, name)) * 31)
    U, I = 3000, 2000
    lr, reg = 0.01, (1e-3, 1e-3)
    recs = []
    if name in ("tiles-small", "tiles-sms"):
        Bs = [1, 63, 64, 65] if name == "tiles-small" else [64 * (sms - 1), 64 * sms, 64 * (sms + 1), 64 * 2 * sms + 37]
        tabs, W = make_problem(rng, U, I, F, L)
        planes = uniform_planes(rng, U, I, sum(Bs))
        st = make(tabs, W, planes, F, L, "sgd", lr, reg, 2 * max(Bs))
        lo = 0
        for B in Bs:
            r = checked_step(st, lo, B, B, f"B={B} {fused_geometry(B, sms)}", ref_device=ref_device)
            r["geometry"] = fused_geometry(B, sms)
            recs.append(r)
            lo += B
        return recs
    if name.startswith("dup-"):
        B = 64 * 40 + 17
        tabs, W = make_problem(rng, U, I, F, L)
        bu, bi, bj = uniform_planes(rng, U, I, 2 * B)
        if name == "dup-user":
            bu[:] = 7
        elif name == "dup-item":
            bi[:] = 11
        else:
            bj[::3] = bi[::3]                                  # i == j: x = 0, the two rows cancel
            bi[1::4], bj[1::4] = bj[0::4][:len(bi[1::4])], bi[0::4][:len(bi[1::4])]   # item pos in one triple, neg in the next
        st = make(tabs, W, (bu, bi, bj), F, L, "sgd", lr, reg, 2 * B)
        recs.append(checked_step(st, 0, B, B, "step 0", ref_device=ref_device))
        recs.append(checked_step(st, B, B, B, "step 1", ref_device=ref_device))
        return recs
    if name == "dead-units":
        B = 64 * 50
        tabs, W = make_problem(rng, U, I, F, L)
        lay = layout(F, L)
        W[lay["b_off"][0]:lay["b_off"][0] + 32] = -50.0      # units 0..31 of layer 1 never fire
        planes = uniform_planes(rng, U, I, B)
        st = make(tabs, W, planes, F, L, "sgd", lr, reg, 2 * B)
        W0 = st.snapshot()["W"]
        r = checked_step(st, 0, B, B, "b1[:32] = -50", ref_device=ref_device)
        W1 = st.snapshot()["W"]
        n0 = widths(F, L)[0]
        r["dead_rows_identical"] = bool(torch.equal(W0[:32 * n0], W1[:32 * n0]) and
                                        torch.equal(W0[lay["b_off"][0]:lay["b_off"][0] + 32], W1[lay["b_off"][0]:lay["b_off"][0] + 32]))
        r["ok"] = r["ok"] and r["dead_rows_identical"]
        recs.append(r)
        return recs
    if name == "saturated":
        B = 64 * 30 + 5
        tabs, W = make_problem(rng, U, I, F, L)
        tabs[0] *= 60.0; tabs[1] *= 60.0                     # |x| reaches 40: the 1e-10 of the BPR coefficient dominates
        planes = uniform_planes(rng, U, I, B)
        st = make(tabs, W, planes, F, L, "sgd", lr, reg, 2 * B)
        r = checked_step(st, 0, B, B, "GMF tables x60", ref_device=ref_device)
        recs.append(r)
        return recs
    if name == "reg0":
        B = 64 * 20 + 3
        tabs, W = make_problem(rng, U, I, F, L)
        planes = uniform_planes(rng, U, I, B)
        st = make(tabs, W, planes, F, L, "sgd", lr, (0.0, 0.0), 2 * B)
        recs.append(checked_step(st, 0, B, B, "reg 0", ref_device=ref_device))
        return recs
    if name == "adam":
        B = 64 * 3 * sms + 9
        tabs, W = make_problem(rng, U, I, F, L)
        planes = uniform_planes(rng, U, I, 3 * B)
        st = make(tabs, W, planes, F, L, "adam", 1e-3, reg, 2 * B)
        for s in range(3):
            recs.append(checked_step(st, s * B, B, B, f"adam step {s}", adam_step0=s, ref_device=ref_device))
        return recs
    if name == "loss-only-65":
        B = 65
        tabs, W = make_problem(rng, U, I, F, L)
        planes = uniform_planes(rng, U, I, B)
        st = make(tabs, W, planes, F, L, "sgd", lr, reg, 2 * B)
        recs.append(checked_step(st, 0, B, B, "apply=False", apply=False, ref_device=ref_device))
        return recs
    if name == "launch-split":
        # one 5-step launch against five 1-step launches (launch_vs_singles).  Wide tables: rows rarely meet in one step, so the
        # two runs' atomics differ in W only, and a W difference of a few fp32 ulps stays inside the noise the reference allows
        # for the next step.
        B, U, I, lr = 64 * 2 * sms + 21, 200_000, 200_000, 1e-4
        tabs, W = make_problem(rng, U, I, F, L)
        planes = uniform_planes(rng, U, I, 5 * B)
        one = make(tabs, W, planes, F, L, "sgd", lr, reg, 2 * B)
        singles = make(tabs, W, planes, F, L, "sgd", lr, reg, 2 * B)
        recs += launch_vs_singles(one, singles, 5 * B, B, 5, ref_device=ref_device)
        return recs
    raise KeyError(name)


def run_layer_case(F, L, make, ref_device, batches=LAYER_BATCHES, tower_dtype=1, mode=0, dropout=0.0):
    plan = tower_plan(tower_dtype, F, L, mode, dropout)
    assert not plan["fused"]
    rng = np.random.default_rng(F * 131 + L * 7 + mode * 3 + int(dropout * 10))
    U, I = 700, 500
    lr, reg = 0.01, (1e-3, 1e-3)
    tabs, W = make_problem(rng, U, I, F, L, mode)
    planes = uniform_planes(rng, U, I, sum(batches))
    recs = []
    st = make(tabs, W, planes, F, L, "sgd", lr, reg, 2 * max(batches), mode=mode, tower_dtype=tower_dtype, dropout=dropout)
    lo = 0
    for s, B in enumerate(batches):
        keep = masks = None
        if dropout > 0:
            keep, words = host_masks(B, F, L, dropout, 100 + s)
            masks = torch.from_numpy(words).to(st.device)
        r = checked_step(st, lo, B, B, f"F={F} L={L} td={tower_dtype} mode={mode} p={dropout} B={B}", keep=keep, masks=masks,
                         ref_device=ref_device)
        r["plan"] = plan
        recs.append(r)
        lo += B
    return recs


def bench_planes(seed, U, I):
    """the bench's index statistics at the ML-20M shape: Zipf-skewed positives, 4 uniform negatives each, one permutation"""
    from daisyrec_b200 import ops
    from daisyrec_b200.utils.synthetic import make_interactions
    d = make_interactions(U, I, 20_000_000, seed=seed, device="cuda")
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    u, i = d["coo_u"].repeat_interleave(4), d["coo_i"].repeat_interleave(4)
    j = torch.randint(0, I, (u.numel(),), generator=g, device="cuda", dtype=torch.int32)
    tr = torch.stack([u, i, j], 1).contiguous()
    del d, u, i, j
    perm = torch.randperm(tr.shape[0], generator=g, device="cuda")
    planes = tuple(x.clone() for x in ops.gather_triples(tr, perm))
    del tr, perm
    return planes


def run_bench_case(make, sms):
    """the bench trajectory (cfg_c3_neumf): ML-20M shape, F = 32, L = 2, Adam lr 1e-3 reg 1e-3, B = 1 048 576 (16 384 tiles)"""
    from daisyrec_b200 import ops
    U, I, F, L, B = 138_493, 26_744, 32, 2, 1 << 20
    planes = bench_planes(2022, U, I)
    T = planes[0].numel()
    D = F << (L - 1)
    g = torch.Generator(device="cuda"); g.manual_seed(11)
    tabs = [(torch.randn(s, device="cuda", generator=g) * 0.05).contiguous() for s in ((U, F), (I, F), (U, D), (I, D))]
    W = (torch.randn(ops.neumf_param_count(F, L), device="cuda", generator=g) * 0.1).contiguous()
    st = make(tabs, W, planes, F, L, "adam", 1e-3, (1e-3, 1e-3), 2 * B)
    nsteps = -(-T // B)
    recs = []

    def add(r):
        r["geometry"] = fused_geometry(r["nb"], sms)
        recs.append(r)

    add(checked_step(st, 0, B, B, "loss only B=1M", apply=False, ref_device="cuda"))
    for s in range(3):
        add(checked_step(st, s * B, B, B, f"step {s}", adam_step0=s, ref_device="cuda"))
    k = nsteps - 2 - 3
    loss = st.run(3 * B, k * B, B, k, adam_step0=3)
    add(dict(tag=f"steps 3..{nsteps - 3} unchecked", nb=k * B, loss=float(loss[-1]), loss_ref=float("nan"), loss_ratio=0.0,
             ratio=0.0, kneed=float("nan"), tensors={}, checks=dict(clean=st.clean()),
             ok=bool(np.all(np.isfinite(loss)) and st.clean())))
    for s in (nsteps - 2, nsteps - 1):
        add(checked_step(st, s * B, min(B, T - s * B), B, f"step {s}", adam_step0=s, ref_device="cuda"))
    return recs


# ---------------------------------------------------------------- GPU tests
def _gpu_make(device="cuda"):
    def make(tabs, W, planes, F, L, opt, lr, reg, max_rows, mode=0, tower_dtype=2, dropout=0.0):
        return GpuNeumf(tabs, W, planes, F, L, opt, lr, reg, max_rows, mode, tower_dtype, dropout, device)
    return make


@pytest.fixture(scope="module")
def gpu():
    from daisyrec_b200 import ops
    ops.require_cuda()
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.gpu
def test_fused_bench_trajectory(gpu):
    sms = gpu
    assert fused_supported(32, 2, 0, 0.0) and fused_geometry(1 << 20, sms)["tiles"] == 16384
    recs = run_bench_case(_gpu_make(), sms)
    assert fused_geometry(1 << 20, sms)["per_cta"] >= 100
    report("bench", recs)
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("name", FUSED_CASES)
def test_fused_step_vs_fp64(gpu, name):
    sms = gpu
    recs = run_fused_case(name, _gpu_make(), sms, "cuda")
    if name == "tiles-sms":
        geo = [r["geometry"] for r in recs]
        assert [x["tiles"] for x in geo] == [sms - 1, sms, sms + 1, 2 * sms + 1]
        assert [x["per_cta"] for x in geo] == [1, 1, 2, 3] and geo[-1]["partial"]
    if name == "tiles-small":
        assert [r["geometry"]["tiles"] for r in recs] == [1, 1, 1, 2]
    report(name, recs)


@pytest.mark.gpu
@pytest.mark.parametrize("F,L", LAYER_SHAPES)
def test_layerwise_bf16_step_vs_fp64(gpu, F, L):
    plan = tower_plan(1, F, L)
    n = widths(F, L)
    assert plan["ig"][0] == (n[0] <= UMMA_MAX_N) and plan["fwd"][0] == (n[1] <= UMMA_MAX_N)
    report(f"layer F={F} L={L}", run_layer_case(F, L, _gpu_make(), "cuda"))


@pytest.mark.gpu
@pytest.mark.parametrize("F,L,tower_dtype,mode,dropout", [(32, 2, 1, 0, 0.5), (12, 2, 1, 0, 0.5), (32, 2, 2, 0, 0.5),
                                                          (32, 2, 1, 2, 0.0), (64, 3, 1, 2, 0.0)])
def test_layerwise_dropout_and_mlp_vs_fp64(gpu, F, L, tower_dtype, mode, dropout):
    plan = tower_plan(tower_dtype, F, L, mode, dropout)
    assert not plan["fused"]                                 # 'fused' under dropout runs the layer-wise bf16 path
    assert plan == tower_plan(1, F, L, mode, dropout)
    report(f"layer F={F} L={L} td={tower_dtype} mode={mode} p={dropout}",
            run_layer_case(F, L, _gpu_make(), "cuda", batches=[64, 2048], tower_dtype=tower_dtype, mode=mode, dropout=dropout))


@pytest.mark.gpu
def test_workspace_carve_mirror(gpu):
    from daisyrec_b200 import _lib
    for opt in ("sgd", "adam"):
        for U, I, F, L in ((700, 500, 32, 2), (13, 7, 12, 3)):
            assert carve(neumf_ws_parts(U, I, F, L, opt))[1] == _lib.lib().drb_neumf_workspace_bytes(U, I, F, L, _lib.OPT_KIND[opt], 0)


def ref_scores(tabs, W, F, L, users, items, plan, mode=0):
    """-> (scores, bound) of the (users[r], items[r]) pairs through the reference forward"""
    UG, IG, UM, IM = (t.to(F64) for t in tabs)
    lay = layout(F, L, mode)
    n = lay["n"]
    Wd = W.to(F64)
    a = torch.cat([UM[users], IM[items]], 1)
    aN = torch.zeros_like(a); aP = torch.zeros_like(a)
    for l in range(L):
        w = Wd[lay["w_off"][l]:lay["w_off"][l] + n[l] * n[l + 1]].view(n[l + 1], n[l])
        b = Wd[lay["b_off"][l]:lay["b_off"][l] + n[l + 1]]
        if plan["fwd"][l]:
            a, aN, aP = rnd(a, aN, aP, Flags(KAPPA)); w = br(w)
        z = a @ w.T + b
        zN = a.abs() @ w.abs().T + b.abs() + aN @ w.abs().T
        zP = aP @ w.abs().T
        live = z > -(KAPPA * U_RND * zN + zP)
        a, aN, aP = torch.relu(z), torch.where(live, zN, 0.0), torch.where(live, zP, 0.0)
    F_ = F
    wp = Wd[lay["wp_off"]:lay["bp_off"]]
    hoff = F_ if mode == 0 else 0
    s = a @ wp[hoff:hoff + F_] + Wd[lay["bp_off"]]
    sN = a.abs() @ wp[hoff:hoff + F_].abs() + aN @ wp[hoff:hoff + F_].abs() + abs(float(Wd[lay["bp_off"]]))
    sP = aP @ wp[hoff:hoff + F_].abs()
    if mode != 2:
        gm = UG[users] * IG[items]
        s = s + gm @ wp[:F_]
        sN = sN + gm.abs() @ wp[:F_].abs()
    return s, KAPPA * U_RND * sN + sP


@pytest.mark.gpu
@pytest.mark.parametrize("F,L", [(32, 2), (64, 3), (12, 2)])
def test_scores_bf16_vs_fp64(gpu, F, L):
    from daisyrec_b200 import ops
    rng = np.random.default_rng(F + L)
    U, I = 300, 700
    tabs, W = make_problem(rng, U, I, F, L)
    tabs_d = [torch.from_numpy(t).cuda() for t in tabs]
    W_d = torch.from_numpy(W).cuda()
    ws = ops.NeumfWorkspace(U, I, F, L, "sgd", 1000, "cuda")           # max_rows 1000: the chunk loop runs
    users = rng.integers(U, size=7).astype(np.int64)
    cands = rng.integers(I, size=(7, 250)).astype(np.int64)
    plan = tower_plan(1, F, L)
    worst = 0.0
    for items, per in ((cands, 250), (None, I)):
        assert len(users) * per > 1000
        sc = {td: ops.neumf_scores(tabs_d, W_d, ws, torch.from_numpy(users).cuda(),
                                   None if items is None else torch.from_numpy(items).cuda(), per, tower_dtype=td) for td in (0, 1, 2)}
        torch.cuda.synchronize()
        uu = torch.from_numpy(np.repeat(users, per)).cuda()
        ii = torch.from_numpy(items.reshape(-1) if items is not None else np.tile(np.arange(I), len(users))).cuda()
        want, bound = ref_scores(tabs_d, W_d, F, L, uu, ii, plan)
        err = (sc[1].reshape(-1).to(F64) - want).abs()
        r = float((err / bound).max())
        worst = max(worst, r)
        assert r <= 1, r
        # tower_dtype 2 scores on the fp32 engine: bit-identical to tower_dtype 0 (DESIGN.md 3.5)
        assert torch.equal(sc[2], sc[0])
        assert not torch.equal(sc[1], sc[0])
    print(f"scores F={F} L={L}: worst error/bound {worst:.3g}")


def second_device_main(out):
    """child: one fused step on cuda:0, then one on cuda:1, each checked against the reference"""
    res = {}
    for dev in ("cuda:0", "cuda:1"):
        torch.cuda.set_device(dev)
        rng = np.random.default_rng(3)
        F, L, U, I, B = 32, 2, 3000, 2000, 64 * 300 + 5
        tabs, W = make_problem(rng, U, I, F, L)
        planes = uniform_planes(rng, U, I, B)
        st = GpuNeumf(tabs, W, planes, F, L, "sgd", 0.01, (1e-3, 1e-3), 2 * B, device=dev)
        r = checked_step(st, 0, B, B, f"fused on {dev}", ref_device=dev)
        print(summary(r), flush=True)
        res[dev] = dict(ok=r["ok"], ratio=r["ratio"])
    with open(out, "w") as f:
        json.dump(res, f)


@pytest.mark.gpu
def test_fused_step_on_second_device(gpu, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU visible")
    out = str(tmp_path / "dev2.json")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "second-device", out], capture_output=True, text=True, timeout=600)
    print(r.stdout[-3000:])
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    with open(out) as f:
        res = json.load(f)
    assert all(v["ok"] for v in res.values()), res


# ---------------------------------------------------------------- CPU checks
def test_bf16_emulation_matches_torch():
    rng = np.random.default_rng(0)
    x = np.concatenate([rng.standard_normal(100_000).astype(np.float32) * 10.0 ** rng.integers(-30, 30, 100_000),
                        np.array([0.0, -0.0, 1e-45, -1e-45, 1e-40, -3e-39, 1.17549435e-38, 3.4e38, -3.4e38, np.inf, -np.inf],
                                 np.float32)]).astype(np.float32)
    # exact ties: the bf16 value plus half its step, with both parities of the kept mantissa bit
    base = (rng.integers(0, 0x7F7F, 2000).astype(np.uint32) << 16)     # finite bf16 values below the largest one
    ties = (base | 0x8000).view(np.float32)
    t = torch.from_numpy(np.concatenate([x, ties, -ties]))
    want = t.to(torch.bfloat16).to(torch.float32)
    got = br(t)
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))
    assert torch.equal(br(t.double()), want.double())


def test_reference_without_rounding_matches_oracle(orc):
    """with every rounding switched off the reference is the fp32 step of the pinned C oracle (regulariser quirk, SGD / Adam with
    bias correction, modes 0 and 2, dropout keep factors)"""
    nr = dict(fused=False, fwd=[False] * 3, wg=[False] * 3, ig=[False] * 3)
    for F, L, mode, opt, drop in ((8, 2, 0, "sgd", 0.0), (12, 3, 0, "adam", 0.0), (8, 2, 2, "sgd", 0.0), (8, 2, 0, "sgd", 0.5),
                                  (8, 2, 2, "adam", 0.5)):
        rng = np.random.default_rng(F + 10 * L + mode)
        U, I, B = 40, 30, 97
        tabs, W = make_problem(rng, U, I, F, L, mode, 0.3, 0.3)
        bu, bi, bj = uniform_planes(rng, U, I, B)
        keep = None
        if drop:
            keep, _ = host_masks(B, F, L, drop, 5)
        reg = (0.002, 0.003)
        lr = 0.05
        to, Wo = [t.copy() for t in tabs], W.copy()
        adam = None if opt == "sgd" else ([np.zeros_like(a) for a in to + [Wo]], [np.zeros_like(a) for a in to + [Wo]])
        lo = orc.neumf_bpr_step(to, Wo, F, L, bu, bi, bj, orc.hyper(lr, reg[0], reg[1], opt), True, adam, 1, mode=mode,
                                keep=None if keep is None else keep.numpy())
        res = ref_step([torch.from_numpy(t) for t in tabs], torch.from_numpy(W), *(torch.from_numpy(x.astype(np.int64)) for x in (bu, bi, bj)),
                       F, L, nr, mode, keep, reg)
        assert abs(res["loss"] - lo) <= 2e-6 * abs(lo), (F, L, mode, opt, res["loss"], lo)
        for k, (t0, want) in enumerate(zip(tabs + [W], to + [Wo])):
            th, g = torch.from_numpy(t0).to(F64).reshape(-1), res["g"][k].reshape(-1)
            if opt == "sgd":
                got = th - lr * g
            else:
                z = torch.zeros_like(th)
                got = adam_apply(th, g, z, z, lr, 1)
            err = (got - torch.from_numpy(want).to(F64).reshape(-1)).abs()
            tol = 2e-6 * max(1.0, float(np.abs(want).max())) if opt == "sgd" else 2e-6
            # Adam: elements whose gradient is fp32 noise of zero take a +-lr step of either sign in the oracle
            noise = (g.abs() < 1e-6) if opt == "adam" else torch.zeros_like(g, dtype=torch.bool)
            assert float(err[~noise].max()) <= tol, (F, L, mode, opt, NAMES[k], float(err[~noise].max()))


def _cpu_problem(seed, B=64 * 3 + 13, F=32, L=2, U=60, I=50):
    rng = np.random.default_rng(seed)
    tabs, W = make_problem(rng, U, I, F, L)
    return tabs, W, uniform_planes(rng, U, I, 3 * B), B


def test_harness_passes_with_fp32_stand_in():
    for F, L, td, opt in ((32, 2, 2, "sgd"), (32, 2, 2, "adam"), (64, 3, 1, "sgd"), (12, 2, 1, "sgd")):
        tabs, W, planes, B = _cpu_problem(F + L, F=F, L=L)
        plan = tower_plan(td, F, L)
        st = StandIn(tabs, W, planes, F, L, opt, 0.01, (1e-3, 1e-3), plan)
        for s in range(2):
            r = checked_step(st, s * B, B, B, f"stand-in {F} {L} {opt} {s}", adam_step0=s)
            assert r["ok"], summary(r)
    # the case plans themselves, with the stand-in playing the device
    mk = lambda tabs, W, planes, F, L, opt, lr, reg, max_rows, mode=0, tower_dtype=2, dropout=0.0: \
        StandIn(tabs, W, planes, F, L, opt, lr, reg, tower_plan(tower_dtype, F, L, mode, dropout), mode)
    for name in ("tiles-small", "dup-mixed", "dead-units"):
        recs = run_fused_case(name, mk, 132, "cpu")
        assert recs and all(r["ok"] for r in recs), [summary(r) for r in recs]


@pytest.mark.parametrize("defect", ["dz1_unrounded", "swap_da0", "drop_tile_gw1", "drop_last_triple", "imj_in_norms", "gb1_rounded"])
@pytest.mark.parametrize("tiles", [3, 301])
def test_harness_flags_defective_stand_in(defect, tiles):
    """each defect fails the harness (error above the bound), on a 3-tile step and on a 301-tile step"""
    B = 64 * (tiles - 1) + 13
    tabs, W, planes, _ = _cpu_problem(7, B=B, U=60 if tiles == 3 else 3000, I=50 if tiles == 3 else 2000)
    assert B % 64 and B > 128
    plan = tower_plan(2, 32, 2)
    reg = (1e-2, 1e-2) if defect == "imj_in_norms" else (1e-3, 1e-3)
    st = StandIn(tabs, W, planes, 32, 2, "sgd", 0.01, reg, plan, defects=(defect,))
    r = checked_step(st, 0, B, B, defect)
    assert not r["ok"], summary(r)
    bad = {k for k, v in r["tensors"].items() if v["ratio"] > 1}
    want = {"dz1_unrounded": {"W1", "UM", "IM"}, "swap_da0": {"UM"}, "drop_tile_gw1": {"W1"}, "drop_last_triple": {"UM", "IM"},
            "imj_in_norms": {"IM"}, "gb1_rounded": {"b1"}}[defect]
    assert bad & want, (defect, bad)
    # the same step without the defect passes
    ok = checked_step(StandIn(tabs, W, planes, 32, 2, "sgd", 0.01, reg, plan), 0, B, B, "no defect")
    assert ok["ok"], summary(ok)


def test_path_mirrors_hand_worked():
    assert fused_supported(32, 2, 0, 0.0)
    assert not fused_supported(32, 2, 0, 0.5) and not fused_supported(64, 2, 0, 0.0) and not fused_supported(32, 3, 0, 0.0)
    assert not fused_supported(32, 2, 2, 0.0)
    assert tower_plan(2, 32, 2)["fused"] and not tower_plan(2, 32, 2, 0, 0.5)["fused"]
    assert tower_plan(2, 32, 2, 0, 0.5) == dict(fused=False, fwd=[True, True], wg=[True, True], ig=[True, True])
    # F = 64, L = 3: widths 512 -> 256 -> 128 -> 64; dA0 = dZ1 W1 has N = 512: fp32
    p = tower_plan(1, 64, 3)
    assert widths(64, 3) == [512, 256, 128, 64]
    assert p["fwd"] == [True, True, True] and p["wg"] == [True, True, True] and p["ig"] == [False, True, True]
    # F = 128, L = 3: widths 1024 -> 512 -> 256 -> 128; the first forward layer (N = 512) is fp32
    p = tower_plan(1, 128, 3)
    assert p["fwd"] == [False, True, True] and p["wg"] == [False, True, True] and p["ig"] == [False, False, True]
    # F = 128, L = 2: N exactly at the 256 cap
    assert tower_plan(1, 128, 2)["fwd"] == [True, True] and tower_plan(1, 128, 2)["ig"] == [False, True]
    assert tower_plan(0, 32, 2) == dict(fused=False, fwd=[False, False], wg=[False, False], ig=[False, False])
    # tile geometry of the fused kernel (one persistent CTA per SM)
    assert fused_geometry(1 << 20, 132) == dict(tiles=16384, grid=132, per_cta=125, partial=False)
    assert fused_geometry(65, 132) == dict(tiles=2, grid=2, per_cta=1, partial=True)
    assert fused_geometry(64 * 264 + 37, 132)["per_cta"] == 3


if __name__ == "__main__":
    if sys.argv[1] == "second-device":
        second_device_main(sys.argv[2])
