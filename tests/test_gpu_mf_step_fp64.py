"""The MF + BPR step of all three instantiations (general, lean, lean user-bucketed in both its forms) against the fp64 oracle.

Teacher forcing: before every checked launch the device tables are copied to the host, oracle.mf_bpr_step (fp64 accumulation)
runs the launch's k <= 4 steps on that copy, and the result is compared element-wise with the device's.  Errors never compound
across launches, so one lost or doubled contribution shows up as one bad launch however long the trajectory.  Per element e
and step, with u = 2^-24 and A_e the sum of |contribution| to e in that step (c (q_i - q_j) for user elements, +-c p_u for item
elements, plus the regulariser terms), computed in numpy fp64 from the oracle's pre-step tables:

    term_e = 2 u |theta_e| + lr (KAPPA u A_e + DELTA)

A single-step launch must meet |gpu - fp64| <= term_e.  In a k-step launch the device starts each later step from its own
tables, which differ from the oracle's by at most the bound E so far.  That difference moves the step's gradient by at most
D_e: its first-order effect through the coefficients (|dc/dx| <= 1/4 times the change of x = p.(q_i - q_j)), through the
partner rows (|c| times their bound) and through the reg_2 term, plus 2 reg_1 per occurrence where the sign of theta is within
the bound.  Each step then sets E <- CARRY (E + lr D) + term on the rows it touches; rows it does not touch keep E, because
neither side moves them.  KAPPA and DELTA were calibrated on the general instantiation (twice its worst ratio) and are the
same for every instantiation and every step of a launch.  Rows that no step of a launch touches must be bit-identical.

The instantiation is chosen once per process, so each runs in child processes (this file run as a script): DRB_NO_LEAN=1
keeps the general kernel, DRB_UBUCKET=0 the plain lean one, DRB_UBUCKET=1 forces the user-bucketed mode wherever it can run.
That mode has two forms, and drb_mf_last_step_staged tells them apart.  Each record's mode is drb_mf_last_step_mode (0
general, 1 lean, 2 user-bucketed), with 3 for the staged SGD form (each bucket's user rows in shared memory, updated when the
bucket completes, batch norms from a per-launch norm cache); 2 is then the accumulate-then-sweep form (Adam, or buckets wider
than the staged rows fit, 84 users at F = 64 and 168 at F = 32).  The cases hit the geometries the
mode runs at (both sides of that width limit at both factor counts, bucket count, buckets per scan thread, partial last
bucket, a bucket count that is not a multiple of the grid, tile boundaries, user runs across tiles, single-user tiles, runs of
one, empty buckets, scratch growth), sized from the SM count of the device.  Every multi-step launch, including 3 steps at the
ML-20M shape, is checked against fp64.  The regulariser-heavy cases (reg_1 = 0.05, reg_2 = 2) make the regulariser at least
10 % of the step on most touched elements, so that a stale batch norm or a regulariser term lost or added per row rather than
per occurrence is far outside the bound; at the default 0.001 such a term is about 1e-8.

The step function of the harness is injectable: the unmarked tests run it on the CPU with the oracle standing in for the
device, and show that the frozen bound sees one dropped or duplicated triple, a triple dropped in step 2 of a 3-step launch,
step 2 run with step 1's batch norms, and one occurrence's regulariser term skipped.

Worst values seen on an H100 80GB HBM3 (132 SMs, 700 W power limit), error / bound and the kappa that alone would be needed:
- single-step launches: 0.991 (nbk-over) in every instantiation; kappa 65 general, 94 lean, 97 bucketed, all at the last
  full step of the ML-20M epoch (the grown tables), at most 13.3 everywhere else;
- multi-step launches: 0.97 / 5.8 general, 0.95 / 6.4 lean, 0.96 / 6.4 bucketed (the 3-step launch at the ML-20M shape: 0.87 /
  5.3 bucketed);
- regulariser-heavy cases: at most 0.77 / 3.9, the regulariser at least 10 % of the gradient on every touched element.
"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

U_RND = 2.0 ** -24
# Calibrated on the general instantiation over every single-step case below (H100 80GB HBM3): the largest kappa any element
# needed was 67.0 (bench shape, last step of the epoch, where the grown tables make the fp32 dot products behind each
# coefficient the least exact; 4.8 - 6.0 in the first steps), hence 2 x 67.  No element needed an error term that A_e does not
# scale (the residual of the smallest steps stays inside 2 u |theta|), hence DELTA = 0.
KAPPA = 134.0
DELTA = 0.0
LOSS_RTOL = 2e-6
# Growth of the error carried into a later step of a launch, on top of its first-order propagation D: a factor of 2 per step
# for what D leaves out (second-order terms, the perturbation of the batch norms; both scale with the square of the carried
# error or with its ratio to the batch's norm, which are below 1e-5 here)
CARRY = 2.0
REG = (0.001, 0.001)            # reg_1, reg_2 of every case but the regulariser-heavy ones
REG_HEAVY = (0.05, 2.0)
REG_SHARE = 0.1                 # regulariser-heavy cases: |regulariser| >= REG_SHARE |gradient| on most touched elements

# ---------------------------------------------------------------- the bucket geometry of the user-bucketed mode
# mirrors ub_users_for / ub_staged in daisyrec_b200/csrc/mf_bpr.cu: about 8 buckets per resident CTA (2 per SM), at least 16
# users, at most what a 64 KB shared accumulator of (F + 1) floats + 1 counter per user holds and kUbMaxRows (512, the keys of
# the per-tile user sort); no bucketing beyond 8 192 buckets (histogram).  The staged SGD form needs two slots of staged rows
# next to the accumulator in 64 KB: width (12 F + 4) bytes.
UB_MIN_USERS, UB_MAX_BUCKETS, UB_MAX_ROWS, CTAS_PER_SM, SCAN_THREADS = 16, 8192, 512, 2, 256
UB_STAGED_SMEM = 65536


def ub_geometry(U, F, batch, sms, opt="sgd"):
    """-> dict(width, nbk, per_thread, partial, bucketed, staged) of the user-bucketed mode for this problem on `sms` SMs"""
    target = 8 * CTAS_PER_SM * sms
    width = min(max(-(-U // target), UB_MIN_USERS), 65536 // ((F + 1) * 4 + 4), UB_MAX_ROWS)
    nbk = -(-U // width)
    bucketed = F in (32, 64) and nbk <= UB_MAX_BUCKETS and batch + 4 * nbk < 2 ** 31
    staged = bucketed and opt == "sgd" and width * (12 * F + 4) <= UB_STAGED_SMEM
    return dict(width=width, nbk=nbk, per_thread=-(-nbk // SCAN_THREADS), partial=U % width != 0, bucketed=bool(bucketed),
                staged=bool(staged))


def expected_mode(inst, variant, geometry):
    """the mode a record reports (GpuStep: 3 staged, 2 accumulate-then-sweep, 1 lean, 0 general) after a launch of
    instantiation `inst` whose user-bucketed geometry (for its optimiser) is given"""
    if inst == "general":
        return 0
    if inst == "lean":
        return variant
    return 3 if geometry["staged"] else 2 if geometry["bucketed"] else 1


# ---------------------------------------------------------------- fp64 reference quantities of one step
def contributions(P, Q, bu, bi, bj, reg1, reg2, signed=False, carry=(), chunk=1 << 17):
    """Per touched row: the sum of |contribution| of the step's triples to each element (and the fp64 gradient if `signed`).
    carry: pairs (EP, EQ) of table-shaped bounds on |device - P|, |device - Q| before the step; for each, the bound (DP, DQ) on
    the change of the step's gradient they cause through the coefficients and the partner rows (the regulariser's share is
    left to the caller: cnt*, lin*).
    -> dict(urows, irows, AP [nu, F], AQ [ni, F], gP, gQ, RP, RQ (|regulariser part|), cntP [nu, 1], cntQ [ni, 1] (occurrences),
            linP, linQ ([n, 1]: d(regulariser) / d(theta) of the reg_2 term), D (list of (DP, DQ)))"""
    from scipy import sparse
    urows, uinv = np.unique(bu, return_inverse=True)
    irows, iinv = np.unique(np.concatenate([bi, bj]), return_inverse=True)
    n, F = len(bu), P.shape[1]
    ii, ij = iinv[:n], iinv[n:]
    AP, AQ = np.zeros((len(urows), F)), np.zeros((len(irows), F))
    gP = np.zeros_like(AP) if signed else None
    gQ = np.zeros_like(AQ) if signed else None
    D = [(np.zeros_like(AP), np.zeros_like(AQ)) for _ in carry]
    s2 = [0.0, 0.0, 0.0]
    for a in range(0, n, chunk):
        b = min(n, a + chunk)
        p = P[bu[a:b]].astype(np.float64)
        qi = Q[bi[a:b]].astype(np.float64)
        qj = Q[bj[a:b]].astype(np.float64)
        s2[0] += float((p * p).sum()); s2[1] += float((qi * qi).sum()); s2[2] += float((qj * qj).sum())
        x = (p * (qi - qj)).sum(1)
        s = 1.0 / (1.0 + np.exp(-x))
        c = -(s * (1.0 - s)) / (1e-10 + s)
        col = np.arange(b - a)
        mat = lambda v, inv, rows: sparse.csr_matrix((v, (inv, col)), shape=(len(rows), b - a))
        su, si, sj = mat(c, uinv[a:b], urows), mat(c, ii[a:b], irows), mat(c, ij[a:b], irows)
        d = qi - qj
        ad, ap = np.abs(d), np.abs(p)
        AP += abs(su) @ ad
        AQ += (abs(si) + abs(sj)) @ ap
        if signed:
            gP += su @ d
            gQ += (si - sj) @ p
        for (EP, EQ), (DP, DQ) in zip(carry, D):
            ep, eqi, eqj = EP[bu[a:b]], EQ[bi[a:b]], EQ[bj[a:b]]
            # c = -(1 - s) up to the 1e-10: |dc/dx| = s (1 - s); x moves by at most |d|.e_p + |p|.(e_qi + e_qj)
            w = s * (1.0 - s) * (ad * ep + ap * (eqi + eqj)).sum(1)
            wu, wi, wj = mat(w, uinv[a:b], urows), mat(w, ii[a:b], irows), mat(w, ij[a:b], irows)
            DP += abs(su) @ (eqi + eqj) + wu @ ad
            DQ += abs(si) @ ep + abs(sj) @ ep + (wi + wj) @ ap
    # regulariser: per occurrence reg1 sgn(theta) + reg2 theta / ||batch rows||_F (the norms couple the whole batch)
    nu, ni, nj = (np.sqrt(v) for v in s2)
    cu = np.bincount(uinv, minlength=len(urows)).astype(np.float64)[:, None]
    ci = np.bincount(ii, minlength=len(irows)).astype(np.float64)[:, None]
    cj = np.bincount(ij, minlength=len(irows)).astype(np.float64)[:, None]
    pu, qr = P[urows].astype(np.float64), Q[irows].astype(np.float64)
    inv = [1.0 / v if v > 0 else 0.0 for v in (nu, ni, nj)]
    RP = cu * (reg1 * (pu != 0) + reg2 * np.abs(pu) * inv[0])
    RQ = ci * (reg1 * (qr != 0) + reg2 * np.abs(qr) * inv[1]) + cj * (reg1 * (qr != 0) + reg2 * np.abs(qr) * inv[2])
    AP += RP
    AQ += RQ
    if signed:
        gP += cu * (reg1 * np.sign(pu) + reg2 * pu * inv[0])
        gQ += ci * (reg1 * np.sign(qr) + reg2 * qr * inv[1]) + cj * (reg1 * np.sign(qr) + reg2 * qr * inv[2])
    return dict(urows=urows, irows=irows, AP=AP, AQ=AQ, gP=gP, gQ=gQ, RP=RP, RQ=RQ, cntP=cu, cntQ=ci + cj,
                linP=reg2 * cu * inv[0], linQ=reg2 * (ci * inv[1] + cj * inv[2]), D=D)


def compare_table(got, ref, rows, E0, E1):
    """Rows outside `rows` must be bit-identical to the reference; rows in it meet the bound E0 + KAPPA E1 (E1: the part KAPPA
    scales; table-shaped).  -> (worst ratio, offending row ids (stray rows first, then the worst first), kappa that alone
    would be needed)."""
    changed = np.nonzero((got != ref).any(1))[0]
    stray = np.setdiff1d(changed, rows)
    g, r = got[rows].astype(np.float64), ref[rows].astype(np.float64)
    e0, e1 = E0[rows], E1[rows]
    err = np.abs(g - r)
    bound = e0 + KAPPA * e1
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(err > 0, err / bound, 0.0)
        need = np.where(e1 > 0, (err - e0) / e1, 0.0)
    rmax = ratio.max(1) if ratio.size else np.zeros(len(rows))
    bad = rows[np.argsort(-rmax, kind="stable")[:int((rmax > 1).sum())]]
    worst = float(rmax.max()) if rmax.size else 0.0
    if len(stray):
        worst = float("inf")
        bad = np.concatenate([stray, bad])
    return worst, bad, float(need.max()) if need.size else 0.0


# ---------------------------------------------------------------- steppers: the device step and its CPU stand-in
class OracleStep:
    """CPU stand-in of the device step: the oracle itself, optionally tampered with to show that the harness sees it:
    tamper(s, bu, bi, bj) -> (bu, bi, bj) rewrites the batch of step s of a launch; post(s, P0, Q0, P, Q, batch, hp) may
    change the tables in place after the oracle has run step s from P0, Q0."""

    def __init__(self, P, Q, planes, opt, lr, tamper=None, post=None):
        from oracle import oracle as orc
        self.orc, self.P, self.Q, self.planes, self.opt, self.lr = orc, P.copy(), Q.copy(), planes, opt, lr
        self.tamper, self.post = tamper, post
        self.adam = tuple(np.zeros_like(a) for a in (P, P, Q, Q)) if opt == "adam" else None

    def tables(self):
        return self.P.copy(), self.Q.copy()

    def batch(self, lo, n):
        return tuple(np.ascontiguousarray(x[lo:lo + n]) for x in self.planes)

    def __call__(self, lo, n, batch, k, reg1, reg2, adam_step0=0):
        hp = self.orc.hyper(self.lr, reg1, reg2, self.opt)
        losses = []
        for s in range(k):
            b = self.batch(lo + s * batch, min(batch, n - s * batch))
            if self.tamper is not None:
                b = self.tamper(s, *b)
            b = [np.ascontiguousarray(x, np.int32) for x in b]
            P0, Q0 = self.tables()
            losses.append(self.orc.mf_bpr_step(self.P, self.Q, *b, hp, True, self.adam, adam_step0 + s + 1)[0])
            if self.post is not None:
                self.post(s, P0, Q0, self.P, self.Q, b, hp)
        return np.array(losses), None

    def workspace_zero(self):
        return True


class GpuStep:
    """The device step (ops.mf_bpr_train_steps) on the current stream or on `stream`; reports which instantiation ran (3 for
    the staged form of the user-bucketed mode)."""

    def __init__(self, P, Q, planes, opt, lr, stream=None):
        import torch
        from daisyrec_b200 import ops
        self.torch, self.ops, self.opt, self.lr, self.stream = torch, ops, opt, lr, stream
        dev = lambda a: a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a)).cuda()
        with torch.cuda.stream(stream) if stream is not None else _null():
            self.P, self.Q = dev(P).clone(), dev(Q).clone()
            self.planes = tuple(dev(x) for x in planes)
            U, I, F = self.P.shape[0], self.Q.shape[0], self.P.shape[1]
            self.ws = ops.MFWorkspace(U, I, F, opt, "cuda")
        torch.cuda.synchronize()

    def tables(self):
        self.torch.cuda.synchronize()
        return self.P.cpu().numpy(), self.Q.cpu().numpy()

    def batch(self, lo, n):
        return tuple(x[lo:lo + n].cpu().numpy() for x in self.planes)

    def __call__(self, lo, n, batch, k, reg1, reg2, adam_step0=0):
        from daisyrec_b200 import _lib as L
        hp = self.ops.hyper(self.lr, reg1, reg2, self.opt)
        with self.torch.cuda.stream(self.stream) if self.stream is not None else _null():
            bu, bi, bj = (x[lo:lo + n] for x in self.planes)
            losses = self.ops.mf_bpr_train_steps(self.P, self.Q, self.ws, bu, bi, bj, batch, 0, k, hp, adam_step0=adam_step0)
            mode = int(L.lib().drb_mf_last_step_mode())
            staged = int(L.lib().drb_mf_last_step_staged())
            assert staged in (0, 1) and (mode == 2 or staged == 0), (mode, staged)
            mode = 3 if staged else mode            # the staged form of the user-bucketed mode
            losses = losses.cpu().numpy()
        self.torch.cuda.synchronize()
        return losses, mode

    def workspace_zero(self):
        """gradient accumulators gP / gQ and row counters cntU / cntI are all zero between launches"""
        import ctypes
        from daisyrec_b200 import _lib as L
        U, I, F = self.P.shape[0], self.Q.shape[0], self.P.shape[1]
        o = (ctypes.c_int64 * 8)()
        L.check(L.lib().drb_mf_workspace_layout(U, I, F, L.OPT_KIND[self.opt], o))
        b = self.ws.buf
        parts = [b[o[6]:o[6] + 4 * U * F], b[o[2]:o[2] + o[3]], b[o[7]:o[7] + 4 * U], b[o[4]:o[4] + o[5]]]
        return sum(int(a.count_nonzero()) for a in parts) == 0


class _null:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


# ---------------------------------------------------------------- the harness
def sgd_launch(st, lo, n, batch, k, lr, reg1, reg2, tag="", share=False):
    """One SGD launch of k <= 4 steps of `st` over planes [lo, lo + n) at launch batch `batch` (the last step may be short),
    checked against k oracle steps run on a host copy of the pre-launch tables (bound: see the module docstring).
    share: also report the fraction of touched elements whose regulariser is at least REG_SHARE of their gradient (worst
    step).  -> record (dict)."""
    from oracle import oracle as orc
    assert 1 <= k <= 4 and (k - 1) * batch < n <= k * batch, (n, batch, k)
    P, Q = st.tables()
    loss, mode = st(lo, n, batch, k, reg1, reg2)
    zero = st.workspace_zero()
    hp = orc.hyper(lr, reg1, reg2, "sgd")
    E0 = [np.zeros(P.shape), np.zeros(Q.shape)]      # bound = E0 + KAPPA E1
    E1 = [np.zeros(P.shape), np.zeros(Q.shape)]
    touched = [np.zeros(len(P), bool), np.zeros(len(Q), bool)]
    lrefs, share_min = [], 1.0
    for s in range(k):
        bu, bi, bj = (np.ascontiguousarray(x, np.int32) for x in st.batch(lo + s * batch, min(batch, n - s * batch)))
        c = contributions(P, Q, bu, bi, bj, reg1, reg2, signed=share, carry=[(E0[0], E0[1]), (E1[0], E1[1])] if s else [])
        pre = (P[c["urows"]].astype(np.float64), Q[c["irows"]].astype(np.float64))
        lrefs.append(orc.mf_bpr_step(P, Q, bu, bi, bj, hp, True, None, 1)[0])        # in place: P, Q = oracle after step s
        for t, T, rows, A in ((0, P, c["urows"], c["AP"]), (1, Q, c["irows"], c["AQ"])):
            touched[t][rows] = True
            e0, e1 = E0[t][rows], E1[t][rows]
            if s:
                (d0, d1) = (c["D"][0][t], c["D"][1][t])
                lin = c["linP" if t == 0 else "linQ"]
                # a sign of theta within the bound may differ on the device: 2 reg_1 per occurrence
                flip = 2 * reg1 * c["cntP" if t == 0 else "cntQ"] * (np.abs(pre[t]) <= e0 + KAPPA * e1)
                e0 = CARRY * (e0 + lr * (d0 + lin * e0 + flip))
                e1 = CARRY * (e1 + lr * (d1 + lin * e1))
            E0[t][rows] = e0 + 2 * U_RND * np.abs(T[rows].astype(np.float64)) + lr * DELTA
            E1[t][rows] = e1 + lr * U_RND * A
        if share:
            for R, g, A in ((c["RP"], c["gP"], c["AP"]), (c["RQ"], c["gQ"], c["AQ"])):
                m = A > 0
                share_min = min(share_min, float((R[m] >= REG_SHARE * np.abs(g[m])).mean()))
    gP, gQ = st.tables()
    rP, badP, kP = compare_table(gP, P, np.nonzero(touched[0])[0], E0[0], E1[0])
    rQ, badQ, kQ = compare_table(gQ, Q, np.nonzero(touched[1])[0], E0[1], E1[1])
    lrefs = np.array(lrefs)
    lrel = float(np.max(np.abs(np.asarray(loss, np.float64) - lrefs) / np.abs(lrefs)))
    rec = dict(tag=tag, kind="sgd", opt="sgd", lo=lo, nb=n, batch=batch, k=k, reg=[reg1, reg2], mode=mode,
               loss=np.asarray(loss).tolist(), loss_ref=lrefs.tolist(), loss_rel=lrel, ratio=max(rP, rQ),
               bad_users=badP[:16].tolist(), bad_items=badQ[:16].tolist(), kappa_need=max(kP, kQ), ws_zero=zero,
               ok=bool(max(rP, rQ) <= 1 and lrel <= LOSS_RTOL and zero))
    if share:
        rec["reg_share"] = share_min
    return rec


def sgd_step(st, lo, nb, batch, lr, tag="", reg=REG):
    """one teacher-forced single-step SGD launch (nb < batch: a short last step)"""
    return sgd_launch(st, lo, nb, batch, 1, lr, *reg, tag=tag)


ADAM_GAIN = 4.0   # |d(m / sqrt v)| <= 4 x the relative gradient error over <= 3 steps (bias-corrected moments of similar weights)


def adam_launches(st, launches, batch, lr, reg1, reg2, tag=""):
    """Adam over <= 3 steps from zero moments: the device's launches [(lo, n, k, adam_step0)] against the oracle's own
    trajectory from the same start, compared after every launch.  Bound per element: the rounding of every step plus lr x
    ADAM_GAIN x the step's relative gradient noise (KAPPA u A_e + DELTA) / |g_e|.  Elements whose fp64 gradient is below its own
    noise bound in any step so far are exempt: Adam turns them into a +-lr step of either sign.  -> records."""
    from oracle import oracle as orc
    P, Q = st.tables()
    adam = tuple(np.zeros_like(a) for a in (P, P, Q, Q))
    acc = [np.zeros(P.shape), np.zeros(Q.shape)]          # accumulated bound
    exempt = [np.zeros(P.shape, bool), np.zeros(Q.shape, bool)]
    rho = [np.zeros(P.shape), np.zeros(Q.shape)]          # running max of the relative gradient noise
    out, step = [], 0
    for lo, n, k, a0 in launches:
        assert a0 == step
        loss, mode = st(lo, n, batch, k, reg1, reg2, adam_step0=a0)
        zero = st.workspace_zero()
        lrefs = []
        for s in range(k):
            bu, bi, bj = (np.ascontiguousarray(x, np.int32) for x in st.batch(lo + s * batch, min(batch, n - s * batch)))
            c = contributions(P, Q, bu, bi, bj, reg1, reg2, signed=True)
            for t, rows, A, g in ((0, c["urows"], c["AP"], c["gP"]), (1, c["irows"], c["AQ"], c["gQ"])):
                noise = KAPPA * U_RND * A + DELTA
                exempt[t][rows] |= (A > 0) & (np.abs(g) <= noise)
                with np.errstate(divide="ignore", invalid="ignore"):
                    rho[t][rows] = np.maximum(rho[t][rows], np.where(A > 0, noise / np.abs(g), 0.0))
            lrefs.append(orc.mf_bpr_step(P, Q, bu, bi, bj, orc.hyper(lr, reg1, reg2, "adam"), True, adam, step + 1)[0])
            for t, T in ((0, P), (1, Q)):
                acc[t] += 2 * U_RND * np.abs(T) + lr * ADAM_GAIN * rho[t]
            step += 1
        gP, gQ = st.tables()
        ratio, bad, nex = 0.0, [], 0
        for t, got, ref in ((0, gP, P), (1, gQ, Q)):
            err = np.abs(got.astype(np.float64) - ref)
            with np.errstate(divide="ignore", invalid="ignore"):
                r = np.where(err > 0, err / acc[t], 0.0)
            r[exempt[t]] = 0.0
            nex += int(exempt[t].sum())
            ratio = max(ratio, float(r.max()))
            bad.append(np.nonzero((r > 1).any(1))[0][:16].tolist())
        lrel = float(np.max(np.abs(loss - np.array(lrefs)) / np.abs(np.array(lrefs))))
        out.append(dict(tag=tag, kind="adam", opt="adam", lo=lo, nb=n, batch=batch, k=k, mode=mode, loss=loss.tolist(),
                        loss_ref=lrefs, loss_rel=lrel, ratio=ratio, bad_users=bad[0], bad_items=bad[1], exempt=nex,
                        ws_zero=zero, ok=bool(ratio <= 1 and lrel <= LOSS_RTOL and zero)))
    return out


# ---------------------------------------------------------------- cases
# Each case: shape (U, I, F, launch batch B) sized from the SM count, the geometry it is built to hit, and a plan run against a
# stepper factory make(P, Q, planes, opt, lr, stream=None).  Planes are int32 (bu, bi, bj).
def tables(rng, U, I, F, scale=0.1):
    return ((rng.standard_normal((U, F)) * scale).astype(np.float32), (rng.standard_normal((I, F)) * scale).astype(np.float32))


def uniform_planes(rng, U, I, n):
    """uniform users and negatives, Zipf-like (squared uniform) positives"""
    return (rng.integers(U, size=n).astype(np.int32), (rng.random(n) ** 2 * I).astype(np.int32),
            rng.integers(I, size=n).astype(np.int32))


STAGED_W = {64: 84, 32: 168}    # the widest staged bucket: width (12 F + 4) <= 65 536


def shape_of(name, sms):
    """-> (U, I, F, B) of a case on a device with `sms` SMs (the numbers in the comments are for 132)"""
    t = 8 * CTAS_PER_SM * sms                # bucket-count target of the width rule (2 112)
    w16 = 16 * t                             # the largest U that still gets the minimum width 16 (33 792)
    return {
        "ml20m": (138_493, 26_744, 64, 1 << 20),                 # the bench: width 66, 2 099 buckets, 9 per scan thread
        "ml20m-f32": (138_493, 26_744, 32, 1 << 20),             # the NCH = 1 geometry
        "width-cap": (600_000 * sms // 132, 26_744, 64, 1 << 20),  # width at its 248 cap: shared accumulator at 64 KB
        "nbk-max": (8192 * 248, 4_000, 64, 1 << 18),             # 8 192 buckets: histogram at 64 KB, 32 per scan thread
        "nbk-over": (8192 * 248 + 1, 4_000, 64, 1 << 18),        # 8 193 buckets: no bucketing (lean kernel)
        "one-bucket": (12, 50, 64, 4096),                        # a single partial bucket
        "exact-multiple": (min(4096, w16), 700, 64, 8192),       # no partial bucket
        "tiles": (3000, 500, 64, 8192),                          # bucket counts at the tile boundaries, short last steps
        "claim": (20_000, 2_000, 64, 1024),                      # 3 nb < (U + I) / 4: claim-mode phase 2
        "scratch": (3000, 500, 64, 65536),                       # scratch growth on two streams
        "multistep": (5000, 700, 64, 8192),                      # a 4-step and a ragged 2-step launch
        "f32-adam": (5000, 700, 32, 8192),
        "f128": (3000, 500, 128, 8192),                          # no bucketed instantiation: the lean kernel runs
        "staged-edge-f64": (84 * t, 4_000, 64, 1 << 16),         # 177 408 users: width 84, the widest staged bucket
        "sweep-edge-f64": (84 * t + 1, 4_000, 64, 1 << 16),      # width 85: accumulate-then-sweep under SGD
        "staged-edge-f32": (168 * t, 4_000, 32, 1 << 16),        # 354 816 users: width 168
        "sweep-edge-f32": (168 * t + 1, 4_000, 32, 1 << 16),     # width 169
        "staged-tail": (84 * (t - 13) + 50, 4_000, 64, 1 << 16),  # width 84, 2 100 buckets (not a multiple of the grid of
                                                                 # 264), the last one 50 users wide
        "runs-f64": (3000, 500, 64, 8192),                       # the user-run boundary patterns, width 16
        "runs-f32": (5000, 700, 32, 8192),
        "reg-staged-f64": (3000, 500, 64, 4096),                 # reg_1 = 0.05, reg_2 = 2 at B = 512 and 4 096
        "reg-staged-f32": (5000, 700, 32, 4096),
        "reg-sweep-f64": (84 * t + 1, 4_000, 64, 4096),          # the same at width 85 / 169: accumulate-then-sweep
        "reg-sweep-f32": (168 * t + 1, 4_000, 32, 4096),
    }[name]


# children: each instantiation runs every case, in two processes (each well inside its timeout)
GPU_GROUPS = [["ml20m", "ml20m-f32", "width-cap", "nbk-max", "nbk-over", "one-bucket", "exact-multiple", "tiles", "claim",
               "scratch", "multistep", "f32-adam", "f128"],
              ["staged-edge-f64", "sweep-edge-f64", "staged-edge-f32", "sweep-edge-f32", "staged-tail", "runs-f64", "runs-f32",
               "reg-staged-f64", "reg-staged-f32", "reg-sweep-f64", "reg-sweep-f32"]]
GPU_CASES = [n for g in GPU_GROUPS for n in g]


def case_reg(name):
    return REG_HEAVY if name.startswith("reg-") else REG


def geometry_misses(name, g, F, sms):
    """the geometry a case is built to hit (`g` for SGD); -> list of what it misses on this device"""
    cap = 65536 // ((F + 1) * 4 + 4)
    sw = STAGED_W.get(F, 0)
    want = {
        "ml20m": dict(bucketed=True, staged=True, partial=True, multi=True, mid=True),
        "ml20m-f32": dict(bucketed=True, staged=True, partial=True, multi=True, mid=True),
        "width-cap": dict(bucketed=True, staged=False, width=cap),
        "nbk-max": dict(bucketed=True, staged=False, width=cap, nbk=UB_MAX_BUCKETS, per_thread=UB_MAX_BUCKETS // SCAN_THREADS,
                        partial=False),
        "nbk-over": dict(bucketed=False, nbk=UB_MAX_BUCKETS + 1),
        "one-bucket": dict(bucketed=True, staged=True, nbk=1, partial=True),
        "exact-multiple": dict(bucketed=True, staged=True, width=UB_MIN_USERS, partial=False),
        "tiles": dict(bucketed=True, staged=True, width=UB_MIN_USERS),
        "claim": dict(bucketed=True, staged=True, width=UB_MIN_USERS),
        "scratch": dict(bucketed=True, staged=True, width=UB_MIN_USERS),
        "multistep": dict(bucketed=True, staged=True, width=UB_MIN_USERS),
        "f32-adam": dict(bucketed=True, width=UB_MIN_USERS),
        "f128": dict(bucketed=False),
        "staged-edge-f64": dict(bucketed=True, staged=True, width=sw, partial=False),
        "sweep-edge-f64": dict(bucketed=True, staged=False, width=sw + 1, partial=True),
        "staged-edge-f32": dict(bucketed=True, staged=True, width=sw, partial=False),
        "sweep-edge-f32": dict(bucketed=True, staged=False, width=sw + 1, partial=True),
        "staged-tail": dict(bucketed=True, staged=True, width=sw, partial=True, ragged_grid=True),
        "runs-f64": dict(bucketed=True, staged=True, width=UB_MIN_USERS),
        "runs-f32": dict(bucketed=True, staged=True, width=UB_MIN_USERS),
        "reg-staged-f64": dict(bucketed=True, staged=True),
        "reg-staged-f32": dict(bucketed=True, staged=True),
        "reg-sweep-f64": dict(bucketed=True, staged=False, width=sw + 1),
        "reg-sweep-f32": dict(bucketed=True, staged=False, width=sw + 1),
    }[name]
    miss = []
    for k, v in want.items():
        if k == "multi":
            ok = g["per_thread"] > 1
        elif k == "mid":
            ok = UB_MIN_USERS < g["width"] < min(cap, sw)
        elif k == "ragged_grid":            # the last round of bucket claims leaves CTAs without a bucket
            ok = g["nbk"] % (CTAS_PER_SM * sms) != 0
        else:
            ok = g[k] == v
        if not ok:
            miss.append(f"{k}: want {v}, geometry {g}")
    return miss


def ml20m_planes(seed, U, I):
    """the bench's index statistics: Zipf-skewed positives of utils.synthetic at the ML-20M shape, 4 uniform negatives each,
    one seeded permutation (80 M triples, on the device)"""
    import torch
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


def run_users(rng, U, B, kind):
    """user planes of one 2-step segment of the runs cases (batch B, two steps):
    hot: user 7 has 30 % of every step, so its run in bucket 0 (users 0..15) crosses two tile boundaries (1 024 records), and
         bucket 2 (users 32..47) never occurs (its rows must stay bit-identical);
    single: the same, and no other user of bucket 0 occurs: its tiles are one run each;
    distinct: B <= U users, each at most once per step (7 919 is prime to U): runs of length 1"""
    k = np.arange(2 * B)
    if kind == "distinct":
        return ((k % B) * 7919 % U).astype(np.int32)
    u = rng.integers(U, size=2 * B)
    u[k % 10 < 3] = 7
    u[(u >= 32) & (u < 48)] += 16
    if kind == "single":
        u[(u < 16) & (u != 7)] += 16
    return u.astype(np.int32)


def run_case(name, make, sms, log=print):
    """Run case `name` against stepper factory `make`; -> list of records (each carries `mode` and `ok`)."""
    U, I, F, B = shape_of(name, sms)
    rng = np.random.default_rng(sum(map(ord, name)) * 7919)
    lr = 0.01
    reg = case_reg(name)
    recs = []

    def add(r):
        recs.extend(r if isinstance(r, list) else [r])
        for x in (r if isinstance(r, list) else [r]):
            log(f"  {name:15s} {x['tag']:22s} nb={x['nb']:>8d} k={x.get('k', 1)} mode={x['mode']} ratio={x['ratio']:.3g} "
                f"loss_rel={x['loss_rel']:.2g}" + (f" kappa_need={x['kappa_need']:.3g}" if "kappa_need" in x else "")
                + (f" reg_share={x['reg_share']:.3f}" if "reg_share" in x else "")
                + ("" if x["ok"] else f"  FAIL users {x['bad_users']} items {x['bad_items']} ws_zero={x['ws_zero']}"))

    if name in ("ml20m", "ml20m-f32"):
        from daisyrec_b200.utils.synthetic import init_tables
        planes = ml20m_planes(2022, U, I)
        T = planes[0].numel()
        P0, Q0 = (x.numpy() for x in init_tables(U, I, F, 2022))
        st = make(P0, Q0, planes, "sgd", lr)
        nsteps = -(-T // B)
        head = 2
        for s in range(head):
            add(sgd_step(st, s * B, B, B, lr, f"step {s}"))
        if name == "ml20m":
            # a 3-step launch against fp64, then an unchecked launch up to the epoch's last two steps (the tables grow, as in
            # the bench), then the last full step and the short last one
            add(sgd_launch(st, head * B, 3 * B, B, 3, lr, *reg, tag=f"steps {head}..{head + 2}"))
            s0 = head + 3
            loss, mode = st(s0 * B, (nsteps - 2 - s0) * B, B, nsteps - 2 - s0, *reg)
            add(dict(tag=f"steps {s0}..{nsteps - 3}", kind="run", opt="sgd", batch=B, nb=(nsteps - 2 - s0) * B, mode=mode,
                     ratio=0.0, loss_rel=0.0, ws_zero=st.workspace_zero(), bad_users=[], bad_items=[],
                     ok=bool(np.all(np.isfinite(loss)) and st.workspace_zero())))
            for s in (nsteps - 2, nsteps - 1):
                add(sgd_step(st, s * B, min(B, T - s * B), B, lr, f"step {s}"))
        return recs
    if name in ("width-cap", "nbk-max", "nbk-over"):
        P0, Q0 = tables(rng, U, I, F)
        planes = uniform_planes(rng, U, I, B)
        st = make(P0, Q0, planes, "sgd", lr)
        add(sgd_step(st, 0, B, B, lr, "step 0"))
        return recs
    if name in ("one-bucket", "exact-multiple", "f32-adam", "f128"):
        P0, Q0 = tables(rng, U, I, F)
        planes = uniform_planes(rng, U, I, 5 * B)
        if name != "f32-adam":
            st = make(P0, Q0, planes, "sgd", lr)
            add(sgd_step(st, 0, B, B, lr, "sgd step 0"))
            add(sgd_step(st, B, B, B, lr, "sgd step 1"))
        st = make(P0, Q0, planes, "adam", lr)
        add(adam_launches(st, [(2 * B, B, 1, 0), (3 * B, 2 * B, 2, 1)], B, lr, *reg, "adam"))
        return recs
    if name == "tiles":
        P0, Q0 = tables(rng, U, I, F)
        # step 0: buckets (width 16) 0, 1, 2 with exactly 1 024, 1 025, 2 048 triples, user 50 (bucket 3) with 3 000, the rest
        # outside buckets 0..4; step 1: all triples in bucket 5; then steps of 1, 3, 4, 5 triples
        u0 = np.concatenate([rng.integers(0, 16, 1024), rng.integers(16, 32, 1025), rng.integers(32, 48, 2048),
                             np.full(3000, 50), rng.integers(80, U, B - 7097)])
        n = 2 * B + 1 + 3 + 4 + 5
        planes = (np.concatenate([u0[rng.permutation(B)], rng.integers(80, 96, B), rng.integers(U, size=13)]).astype(np.int32),
                  (rng.random(n) ** 2 * I).astype(np.int32), rng.integers(I, size=n).astype(np.int32))
        st = make(P0, Q0, planes, "sgd", lr)
        add(sgd_step(st, 0, B, B, lr, "1024/1025/2048/3000"))
        add(sgd_step(st, B, B, B, lr, "one bucket"))
        lo = 2 * B
        for k in (1, 3, 4, 5):
            add(sgd_step(st, lo, k, B, lr, f"short nb={k}"))
            lo += k
        return recs
    if name == "claim":
        P0, Q0 = tables(rng, U, I, F)
        planes = uniform_planes(rng, U, I, 3 * B)
        st = make(P0, Q0, planes, "sgd", lr)
        for s in range(3):
            add(sgd_step(st, s * B, B, B, lr, f"step {s}"))
        return recs
    if name == "scratch":
        # launch batches 4 096 -> 65 536 -> 4 096 (the scratch grows once, then is reused), on the default stream and then on a
        # second stream with its own scratch
        import torch
        P0, Q0 = tables(rng, U, I, F)
        small = 4096
        planes = uniform_planes(rng, U, I, 2 * (2 * small + B))
        for which, stream in (("default", None), ("side", torch.cuda.Stream() if torch.cuda.is_available() else None)):
            st = make(P0, Q0, planes, "sgd", lr, stream=stream)
            lo = 0 if which == "default" else 2 * small + B
            for b in (small, B, small):
                add(sgd_step(st, lo, b, b, lr, f"{which} B={b}"))
                lo += b
        return recs
    if name == "multistep":
        # a 4-step launch and a 2-step launch with a short last step, each against 4 / 2 fp64 steps from its host copy
        P0, Q0 = tables(rng, U, I, F)
        planes = uniform_planes(rng, U, I, 6 * B)
        st = make(P0, Q0, planes, "sgd", lr)
        add(sgd_launch(st, 0, 4 * B, B, 4, lr, *reg, tag="4-step launch"))
        add(sgd_launch(st, 4 * B, B + 3001, B, 2, lr, *reg, tag="2-step, short last"))
        return recs
    if name in ("staged-edge-f64", "sweep-edge-f64", "staged-edge-f32", "sweep-edge-f32", "staged-tail"):
        # a single step, then a 2-step launch with a short last step (most buckets hold 15 - 30 triples of a step)
        P0, Q0 = tables(rng, U, I, F)
        planes = uniform_planes(rng, U, I, 3 * B)
        st = make(P0, Q0, planes, "sgd", lr)
        add(sgd_step(st, 0, B, B, lr, "step 0"))
        add(sgd_launch(st, B, B + 777, B, 2, lr, *reg, tag="2-step, short last"))
        return recs
    if name in ("runs-f64", "runs-f32"):
        # 2-step launches of the user-run patterns (run_users), then a 3-step launch with a short last step, and the hot
        # pattern without a regulariser (no norm cache)
        P0, Q0 = tables(rng, U, I, F)
        bd = 2048                             # runs of one: B <= U
        segs = [("hot", B, 2 * B), ("single", B, 2 * B), ("distinct", bd, 2 * bd)]
        us = [run_users(rng, U, b, kind) for kind, b, _ in segs]
        us.append(rng.integers(U, size=2 * B + 1000).astype(np.int32))
        us.append(run_users(rng, U, B, "hot"))
        u = np.concatenate(us)
        n = len(u)
        planes = (u, (rng.random(n) ** 2 * I).astype(np.int32), rng.integers(I, size=n).astype(np.int32))
        st = make(P0, Q0, planes, "sgd", lr)
        lo = 0
        for kind, b, m in segs:
            add(sgd_launch(st, lo, m, b, 2, lr, *reg, tag=f"{kind} B={b}"))
            lo += m
        add(sgd_launch(st, lo, 2 * B + 1000, B, 3, lr, *reg, tag="3-step, short last"))
        lo += 2 * B + 1000
        add(sgd_launch(st, lo, 2 * B, B, 2, lr, 0.0, 0.0, tag="hot, no regulariser"))
        return recs
    if name.startswith("reg-"):
        # regulariser-heavy: 2-step launches at B = 512 and 3-step launches at B = 4 096
        P0, Q0 = tables(rng, U, I, F)
        planes = uniform_planes(rng, U, I, 2 * 512 + 3 * B)
        st = make(P0, Q0, planes, "sgd", lr)
        add(sgd_launch(st, 0, 2 * 512, 512, 2, lr, *reg, tag="B=512", share=True))
        add(sgd_launch(st, 2 * 512, 3 * B, B, 3, lr, *reg, tag=f"B={B}", share=True))
        return recs
    raise KeyError(name)


# ---------------------------------------------------------------- child process: one instantiation, a group of cases
INSTANTIATIONS = {"general": {"DRB_NO_LEAN": "1"}, "lean": {"DRB_UBUCKET": "0"}, "bucketed": {"DRB_UBUCKET": "1"}}


def child_main(out, cases):
    import traceback
    import torch
    from daisyrec_b200 import _lib as L, ops
    ops.require_cuda()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    res = dict(sms=sms, cases={})

    def make(P, Q, planes, opt, lr, stream=None):
        return GpuStep(P, Q, planes, opt, lr, stream)

    for name in cases:
        t0 = time.time()
        U, I, F, B = shape_of(name, sms)
        try:
            recs = run_case(name, make, sms)
            err = None
        except Exception:
            recs, err = [], traceback.format_exc()
            print(err, flush=True)
        res["cases"][name] = dict(U=U, I=I, F=F, B=B, geometry=ub_geometry(U, F, B, sms), records=recs, error=err,
                                  variant=int(L.lib().drb_mf_step_variant(F, U + I, None, None)), seconds=time.time() - t0)
        torch.cuda.empty_cache()
        print(f"[{name}] {time.time() - t0:.1f} s", flush=True)
    with open(out, "w") as f:
        json.dump(res, f, default=lambda o: o.item() if hasattr(o, "item") else str(o))


def auto_main():
    """no switch: which instantiation the on-device selection runs at the bench shape (printed, not asserted: it is timed)"""
    import torch
    from daisyrec_b200 import _lib as L, ops
    U, I, F, B = shape_of("ml20m", 0)
    rng = np.random.default_rng(1)
    P0, Q0 = tables(rng, U, I, F, 0.01)
    st = GpuStep(P0, Q0, uniform_planes(rng, U, I, B), "sgd", 0.01)
    _, mode = st(0, B, B, 1, *REG)
    print(f"selection at the bench shape: mode {mode} (variant {L.lib().drb_mf_step_variant(F, U + I, None, None)}, "
          f"ms general / lean {ops.mf_step_selfcheck_ms(F, U + I)[:2]})", flush=True)
    assert torch.cuda.is_available()


# ---------------------------------------------------------------- GPU tests
_RESULTS = {}


def _child(tmp_path_factory, inst, group):
    key = (inst, group)
    if key not in _RESULTS:
        out = str(tmp_path_factory.mktemp("fp64") / f"{inst}-{group}.json")
        env = dict(os.environ)
        env.pop("DRB_UBUCKET", None)
        env.pop("DRB_NO_LEAN", None)
        env.update(INSTANTIATIONS[inst])
        t0 = time.time()
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "child", out] + GPU_GROUPS[group], env=env,
                           capture_output=True, text=True, timeout=1200)
        print(r.stdout[-8000:])
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
        with open(out) as f:
            _RESULTS[key] = json.load(f)
        print(f"{inst} / group {group}: child {time.time() - t0:.1f} s")
    return _RESULTS[key]


@pytest.mark.gpu
@pytest.mark.parametrize("inst", list(INSTANTIATIONS))
@pytest.mark.parametrize("name", GPU_CASES)
def test_step_vs_fp64(tmp_path_factory, name, inst):
    group = next(k for k, g in enumerate(GPU_GROUPS) if name in g)
    res = _child(tmp_path_factory, inst, group)
    sms = res["sms"]
    c = res["cases"][name]
    assert c["error"] is None, c["error"]
    g = c["geometry"]
    assert not geometry_misses(name, g, c["F"], sms), geometry_misses(name, g, c["F"], sms)
    # the lean child runs the lean kernel where the on-device selection chose it (it is timed against the general one, which
    # stays where the lean one is not 2 % faster: F = 32 on an H100); the bucketed child runs the bucketed mode wherever it can,
    # in the staged form under SGD where the bucket's rows fit, in the accumulate-then-sweep form otherwise
    if inst == "lean":
        assert c["variant"] in (0, 1)
    recs = c["records"]
    assert recs
    worst = max(r["ratio"] for r in recs)
    need = max((r.get("kappa_need", 0.0) for r in recs), default=0.0)
    modes = sorted({r["mode"] for r in recs})
    print(f"{name} / {inst}: geometry {g}; selection {c['variant']}; modes {modes}; worst error/bound {worst:.3g}, "
          f"kappa_need {need:.3g} over {len(recs)} launches")
    for r in recs:
        want = expected_mode(inst, c["variant"], ub_geometry(c["U"], c["F"], r["batch"], sms, r["opt"]))
        assert r["mode"] == want, (r["tag"], r["mode"], want)
        assert r["ok"], r
        if name.startswith("reg-"):         # the regulariser is a visible part of the step
            assert r["reg_share"] >= 0.5, r


@pytest.mark.gpu
def test_selection_at_bench_shape_is_reported():
    env = dict(os.environ)
    env.pop("DRB_UBUCKET", None)
    env.pop("DRB_NO_LEAN", None)
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "auto"], env=env, capture_output=True, text=True, timeout=600)
    print(r.stdout)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert "selection at the bench shape: mode" in r.stdout


# ---------------------------------------------------------------- CPU checks of the harness itself
def _oracle_make(tamper=None, post=None):
    def make(P, Q, planes, opt, lr, stream=None):
        return OracleStep(P, Q, planes, opt, lr, tamper, post)
    return make


def _small_case(B=2048, steps=3):
    rng = np.random.default_rng(5)
    U, I, F = 300, 200, 64
    P0, Q0 = tables(rng, U, I, F)
    return rng, U, I, F, B, P0, Q0, uniform_planes(rng, U, I, steps * B)


def test_harness_passes_with_oracle_stand_in():
    rng, U, I, F, B, P0, Q0, planes = _small_case()
    st = OracleStep(P0, Q0, planes, "sgd", 0.01)
    recs = [sgd_step(st, 0, B, B, 0.01), sgd_step(st, B, B - 5, B, 0.01)]
    st = OracleStep(P0, Q0, planes, "sgd", 0.01)
    recs += [sgd_launch(st, 0, 3 * B - 5, B, 3, 0.01, *REG), sgd_launch(st, 0, 2 * B, B, 2, 0.01, *REG_HEAVY)]
    st = OracleStep(P0, Q0, planes, "adam", 0.01)
    recs += adam_launches(st, [(0, B, 1, 0), (B, 2 * B, 2, 1)], B, 0.01, *REG)
    assert all(r["ok"] for r in recs), recs
    assert all(r["kappa_need"] <= 0 for r in recs if "kappa_need" in r)   # the oracle against itself: no error at all
    for name in ("one-bucket", "tiles", "multistep", "runs-f64", "reg-staged-f64", "reg-staged-f32"):   # the case plans
        recs = run_case(name, _oracle_make(), 132, log=lambda s: None)
        assert recs and all(r["ok"] for r in recs), (name, recs)
        if name.startswith("reg-"):        # what the GPU test asserts of these cases holds of the plans themselves
            assert all(r["reg_share"] >= 0.5 for r in recs), [r["reg_share"] for r in recs]


def test_runs_cases_cover_the_sort_boundaries():
    """the hot user holds more than two and at most three index tiles (1 024 records) of a step, bucket 2 never occurs, the
    single-user tiles hold no other user of bucket 0, and the runs of one never repeat a user within a step"""
    for name in ("runs-f64", "runs-f32"):
        U, I, F, B = shape_of(name, 132)
        rng = np.random.default_rng(0)
        for kind in ("hot", "single"):
            u = run_users(rng, U, B, kind)
            for s in range(2):
                us = u[s * B:(s + 1) * B]
                assert 2048 < int((us == 7).sum()) <= 3 * 1024 - 16, (name, kind)
                assert not ((us >= 32) & (us < 48)).any()
                if kind == "single":
                    assert set(us[us < 16].tolist()) == {7}
        u = run_users(rng, U, 2048, "distinct")
        assert all(np.unique(u[s * 2048:(s + 1) * 2048]).size == 2048 for s in range(2))


def _typical_triple(planes, B, lo=0):
    """a triple of the step at `lo` whose user occurs 2..64 times in the step and whose coefficient is not negligible"""
    bu = planes[0][lo:lo + B]
    cnt = np.bincount(bu)
    t = int(np.nonzero((cnt[bu] >= 2) & (cnt[bu] <= 64))[0][0])
    return t, int(bu[t]), int(cnt[bu[t]])


@pytest.mark.parametrize("how", ["drop", "duplicate"])
def test_harness_sees_one_lost_or_doubled_contribution(how):
    rng, U, I, F, B, P0, Q0, planes = _small_case()
    t, user, n_user = _typical_triple(planes, B)
    assert n_user <= 64

    def tamper(s, bu, bi, bj):
        if len(bu) != B or not (bu[t] == planes[0][t] and bi[t] == planes[1][t]):
            return bu, bi, bj
        if how == "drop":
            return tuple(np.delete(x, t) for x in (bu, bi, bj))
        return tuple(np.append(x, x[t]) for x in (bu, bi, bj))

    st = OracleStep(P0, Q0, planes, "sgd", 0.01, tamper)
    r = sgd_step(st, 0, B, B, 0.01)
    assert not r["ok"] and r["ratio"] > 1
    assert user in r["bad_users"], r
    assert {int(planes[1][t]), int(planes[2][t])} & set(r["bad_items"]), r
    # the untampered step that follows passes again (teacher forcing: one bad step stays one bad step)
    r2 = sgd_step(st, B, B, B, 0.01)
    assert r2["ok"], r2


def _norms(P, Q, b):
    """inverse batch norms (u, i, j) of batch b on tables P, Q, as the step derives them"""
    return [1.0 / np.sqrt((T[x].astype(np.float64) ** 2).sum()) for T, x in ((P, b[0]), (Q, b[1]), (Q, b[2]))]


@pytest.mark.parametrize("how", ["drop-in-step-2", "stale-norms", "skip-one-regulariser"])
def test_multistep_bound_sees_a_fault_in_a_later_step(how):
    """A 3-step launch of the regulariser-heavy configuration at B = 512: untampered it passes; it fails when step 2 loses one
    triple, when step 2 runs with step 1's batch norms (a norm cache that was not rewritten), and when one occurrence's
    regulariser term is left out of step 2."""
    B, lr = 512, 0.01
    reg1, reg2 = REG_HEAVY
    rng, U, I, F, B, P0, Q0, planes = _small_case(B, 3)
    t, user, _ = _typical_triple(planes, B, lo=B)         # a triple of step 2 (index 1 in the launch)
    item = int(planes[1][B + t])
    seen = {}

    def tamper(s, bu, bi, bj):
        if how == "drop-in-step-2" and s == 1:
            return tuple(np.delete(x, t) for x in (bu, bi, bj))
        return bu, bi, bj

    def post(s, P0_, Q0_, P, Q, b, hp):
        inv = _norms(P0_, Q0_, b)
        if s == 0:
            seen["inv"] = inv
        if s != 1:
            return
        if how == "stale-norms":             # step 2's reg_2 term with step 1's inverse norms instead of its own
            for T, T0, x, k in ((P, P0_, b[0], 0), (Q, Q0_, b[1], 1), (Q, Q0_, b[2], 2)):
                rows, cnt = np.unique(x, return_counts=True)
                T[rows] = (T[rows] + lr * reg2 * cnt[:, None] * T0[rows].astype(np.float64)
                           * (inv[k] - seen["inv"][k])).astype(np.float32)
        elif how == "skip-one-regulariser":   # the positive item of one triple loses that occurrence's regulariser
            q = Q0_[item].astype(np.float64)
            Q[item] = (Q[item] + lr * (reg1 * np.sign(q) + reg2 * q * inv[1])).astype(np.float32)

    ok = sgd_launch(OracleStep(P0, Q0, planes, "sgd", lr), 0, 3 * B, B, 3, lr, reg1, reg2)
    assert ok["ok"], ok
    r = sgd_launch(OracleStep(P0, Q0, planes, "sgd", lr, tamper, post), 0, 3 * B, B, 3, lr, reg1, reg2)
    assert not r["ok"] and r["ratio"] > 1, r
    if how == "drop-in-step-2":
        assert user in r["bad_users"], r
    elif how == "skip-one-regulariser":
        assert item in r["bad_items"], r
    else:
        assert len(r["bad_users"]) >= 16 and len(r["bad_items"]) >= 16, r


def test_geometry_mirror_hand_computed():
    # 132 SMs: 16 x 132 = 2 112 users per width unit; cap 248 at F = 64 (65 536 // 264), 481 at F = 32; staged up to 84 users
    # per bucket at F = 64 (84 x 772 = 64 848 B, 85 x 772 = 65 620 B) and 168 at F = 32 (168 x 388 = 65 184 B, 169: 65 572 B)
    G = lambda U, F=64, B=1 << 20, sms=132, opt="sgd": ub_geometry(U, F, B, sms, opt)
    assert G(138_493) == dict(width=66, nbk=2099, per_thread=9, partial=True, bucketed=True, staged=True)
    assert G(138_493, 32) == dict(width=66, nbk=2099, per_thread=9, partial=True, bucketed=True, staged=True)
    assert G(138_493, opt="adam") == dict(width=66, nbk=2099, per_thread=9, partial=True, bucketed=True, staged=False)
    assert G(600_000) == dict(width=248, nbk=2420, per_thread=10, partial=True, bucketed=True, staged=False)
    assert G(2_031_616, B=1 << 18) == dict(width=248, nbk=8192, per_thread=32, partial=False, bucketed=True, staged=False)
    assert G(2_031_617, B=1 << 18) == dict(width=248, nbk=8193, per_thread=33, partial=True, bucketed=False, staged=False)
    assert G(12, B=4096) == dict(width=16, nbk=1, per_thread=1, partial=True, bucketed=True, staged=True)
    assert G(4096, B=8192) == dict(width=16, nbk=256, per_thread=1, partial=False, bucketed=True, staged=True)
    assert G(3000, 128, 8192)["bucketed"] is False and G(3000, 128, 8192)["staged"] is False
    assert G(33_792)["width"] == 16 and G(33_793)["width"] == 17
    assert G(138_493, sms=114)["width"] == 76                    # 1 824 users per width unit on a 114-SM part
    # the staged width limit, both sides, at both factor counts, on 132 and on 114 SMs (1 824 users per width unit)
    for sms, t in ((132, 2112), (114, 1824)):
        assert G(84 * t, sms=sms) == dict(width=84, nbk=t, per_thread=-(-t // 256), partial=False, bucketed=True, staged=True)
        assert G(84 * t + 1, sms=sms)["width"] == 85 and G(84 * t + 1, sms=sms)["staged"] is False
        assert G(84 * t + 1, sms=sms)["bucketed"] is True
        assert G(168 * t, 32, sms=sms) == dict(width=168, nbk=t, per_thread=-(-t // 256), partial=False, bucketed=True,
                                               staged=True)
        assert G(168 * t + 1, 32, sms=sms)["width"] == 169 and G(168 * t + 1, 32, sms=sms)["staged"] is False
        assert G(168 * t + 1, 32, sms=sms)["bucketed"] is True
        assert G(84 * t, sms=sms, opt="adam")["staged"] is False
    assert (G(177_408)["width"], G(177_409)["width"], G(354_816, 32)["width"], G(354_817, 32)["width"]) == (84, 85, 168, 169)
    # kUbMaxRows: below F = 31 the accumulator would hold more than the 512 keys of the tile sort
    assert G(10 ** 7, 16, sms=132)["width"] == 512 and G(10 ** 7, 28, sms=132)["width"] == 512
    assert G(10 ** 7, 31, sms=132)["width"] == 65536 // 132
    # every case hits its target at 132 SMs and at 114
    for sms in (132, 114):
        for name in GPU_CASES:
            U, I, F, B = shape_of(name, sms)
            assert not geometry_misses(name, ub_geometry(U, F, B, sms), F, sms), (name, sms)
    # both sides of the staged width limit at both factor counts are among the cases
    for sms in (132, 114):
        sides = set()
        for name in GPU_CASES:
            U, I, F, B = shape_of(name, sms)
            g = ub_geometry(U, F, B, sms)
            if g["width"] in (STAGED_W.get(F), STAGED_W.get(F, 0) + 1):
                sides.add((F, g["staged"]))
        assert sides == {(64, True), (64, False), (32, True), (32, False)}, sms


if __name__ == "__main__":
    if sys.argv[1] == "child":
        child_main(sys.argv[2], sys.argv[3:])
    else:
        auto_main()
