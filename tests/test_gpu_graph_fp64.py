"""The LightGCN + BPR and NGCF + BPR steps (segmented SpMM, the MF step's phases 1 and 2, NGCF's BiGNN GEMMs in fp32 and bf16)
against float64 references, one teacher-forced step at a time (fp64_step.py: the snapshot, the bound and its checks).  The
moments are read from the workspace through a mirror of carve_lgcn / carve_ngcf.

References.  `lgcn_ref`: E_mean = 1/(L+1) sum_l A^l E0, BPR on E_mean (gamma = 1e-10), the un-squared L1 / Frobenius
regulariser on the EGO rows counted per occurrence, backward = the same propagation of dL/dE_mean.  `ngcf_ref`: per layer
X = A E, [S | T] = [E + X | X * E], y = S W1^T + b1 + T W2^T + b2, z = LeakyReLU_0.2(y), E' = z / max(||z||, 1e-12); scores on
cat(E_0 .. E_L), the same regulariser on the ego rows, the normalise / LeakyReLU backward of ngcf_act_bwd_kernel.  With
tower_dtype 1 every BiGNN GEMM (N <= 256 always holds) rounds its two operands to bf16 (emulated from the fp32 bits).
`ngcf_ref` also takes one forward's dropout masks (message keep bytes, node keep bytes over the CSR slots with
RefGraph.dropped_by); without them it is the reference above, unchanged.  test_gpu_ngcf_dropout_fp64.py runs the dropout
cases.

N_e runs the chain on |E|, |W|, |G| (A is non-negative).  P_e: LightGCN has none (its bound is pure KAPPA); NGCF has
LeakyReLU gates whose pre-activation lies within its noise of 0 (slope 1 against 0.2 in the backward) and, in bf16, operands
within their noise of a rounding midpoint; the flagged intermediates must stay under PHI_FRAC_MAX.  Under SGD the elements
with no contribution are, for LightGCN, the nodes more than L hops from every batch row, for NGCF the W sections nothing
reaches.
"""
import math
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)
import fp64_step  # noqa: E402
from fp64_step import (F64, GAMMA, KAPPA_LADDER, U_RND, Flags, Stepper, _A, adam_apply, br, carve, checked_step,  # noqa: E402
                       device_tensor, launch_vs_singles, mm, report, rnd, summary, views)

# Calibrated on one H100 80GB HBM3 (700 W power limit) over every GPU case below; the whole file runs in 70 s there.
# "Needed" is the per-element KAPPA of an SGD step where P_e = 0, else (Adam, bf16, the forward) the smallest KAPPA of
# KAPPA_LADDER at which every element of the step passes; the ladder starts at 0.125.
#   LightGCN: 10.6, at E0[3013, 21] of the duplicated-triples step of test_lgcn_launches (bench shape: 0.24 under SGD at
#     E0 elements of both checked steps, <= 0.5 under Adam), hence 24.  Worst error/bound: 0.40 - 0.46 on the bench
#     trajectory, 0.49 on the launches, <= 0.073 on the SpMM geometry (F = 1024).
#   NGCF fp32: steps 0.019 (E0[70824, 12], bench shape, SGD step 1; <= 0.125 elsewhere), the forward 1.5 (bench widths and
#     [256, 256]), hence 3.  Worst error/bound <= 0.49 on the steps (W2[2][2196] at the bench shape), 0.80 under Adam at the
#     bench shape, <= 0.47 on the forward.
#   NGCF bf16: steps 0.5 ([64, 10], [6, 6], [256, 256] and the bench shape under SGD), the forward 1.5 (bench widths,
#     [256, 256]), hence 3.  At KAPPA 3 at most 21 % of the rounded or gated intermediates of a step are flagged
#     ([16, 24, 10, 6, 8]; 19 % at the bench widths, 0.9 - 12 % elsewhere), hence the 40 % ceiling.  Worst error/bound 1.00
#     (elements that need P_e), 0.997 on the forward.  Each bf16 operand (S, T, W1, W2, dY) left unrounded in one layer is
#     caught at 17x - 1600x the bound (test_harness_flags_defective_stand_in).
KAPPA = {"lgcn": 24.0, "ngcf": 3.0, "ngcf_bf16": 3.0}
PHI_FRAC_MAX = 0.4
UMMA_MAX_N = 256


def kappa_of(model, tower_dtype=0):
    return KAPPA["ngcf_bf16"] if model == "ngcf" and tower_dtype == 1 else KAPPA[model]


# ---------------------------------------------------------------- mirror of umma_stage_tile's 16-byte predicate
def stage_vec_loads(base, ld, mn_major, rows, K, fixed=True):
    """byte addresses of the 16-byte loads umma_stage_tile issues for one operand, over its first two K chunks and first 16
    rows (row r0 = 0; the other row tiles start at multiples of 128).  K-major: src(r, k) = S[r ld + k], MN-major:
    src(r, k) = S[k ld + r].  fixed: the predicate with the base-pointer check, else the one before it (ld % 4 == 0 only)."""
    if ld % 4 or (fixed and base % 16):
        return []
    out = []
    for k0 in range(0, min(K, 64), 32):
        if not mn_major:
            out += [base + 4 * (r * ld + k0 + 8 * c) for r in range(min(rows, 16)) for c in range(4) if k0 + 8 * c + 8 <= K]
        else:
            out += [base + 4 * ((k0 + c) * ld + r) for r in range(0, min(rows, 16), 8) for c in range(32)
                    if k0 + c < K and r + 8 <= rows and r % 4 == 0]
    return out


def ngcf_gemm_operands(dims, ws_base=0, w_base=0, n=1000):
    """the operands umma_stage_tile stages for NGCF's six GEMMs per layer (ngcf.cu): (site, base bytes, ld, mn_major, rows, K).
    ST, dY: 256-byte aligned workspace slices; W: the parameter block."""
    out, o = [], 0
    for l in range(len(dims) - 1):
        i, p = dims[l], dims[l + 1]
        W1, W2 = w_base + 4 * o, w_base + 4 * (o + i * p + p)
        S, T, dY = ws_base, ws_base + 4 * i, ws_base
        out += [(f"L{l} fwd1 A", S, 2 * i, False, n, i), (f"L{l} fwd1 B", W1, i, False, p, i),
                (f"L{l} fwd2 A", T, 2 * i, False, n, i), (f"L{l} fwd2 B", W2, i, False, p, i),
                (f"L{l} wg1 A", S, 2 * i, True, i, n), (f"L{l} wg1 B", dY, p, True, p, n),
                (f"L{l} wg2 A", T, 2 * i, True, i, n), (f"L{l} wg2 B", dY, p, True, p, n),
                (f"L{l} ig1 A", dY, p, False, n, p), (f"L{l} ig1 B", W1, i, True, i, p),
                (f"L{l} ig2 A", dY, p, False, n, p), (f"L{l} ig2 B", W2, i, True, i, p)]
        o += 2 * (i * p + p)
    return out


def neumf_gemm_operands(F, L, ws_base=0, w_base=0, n=1000):
    """the same for the NeuMF tower's layer-wise GEMMs (neumf.cu): widths 2D >> l, W_l then b_l per layer"""
    D = F << (L - 1)
    w = [2 * D >> l for l in range(L + 1)]
    out, o = [], 0
    for l in range(L):
        Wl = w_base + 4 * o
        out += [(f"L{l} fwd A", ws_base, w[l], False, n, w[l]), (f"L{l} fwd B", Wl, w[l], False, w[l + 1], w[l]),
                (f"L{l} wg A", ws_base, w[l], True, w[l], n), (f"L{l} wg B", ws_base, w[l + 1], True, w[l + 1], n),
                (f"L{l} ig A", ws_base, w[l + 1], False, n, w[l + 1]), (f"L{l} ig B", Wl, w[l], True, w[l], w[l + 1])]
        o += w[l] * w[l + 1] + w[l + 1]
    return out


# ---------------------------------------------------------------- graphs
class RefGraph:
    """A_hat as float64 (and float32) sparse CSR on `device`, plus the row structure"""

    def __init__(self, row_ptr, col, val, device="cpu"):
        rp = torch.as_tensor(np.asarray(row_ptr, np.int64))
        cl = torch.as_tensor(np.asarray(col, np.int64))
        vl = torch.as_tensor(np.asarray(val, np.float32))
        self.n = len(rp) - 1
        self.row_ptr, self.col, self.val = rp, cl, vl
        self.device = device
        self.A = {dt: torch.sparse_csr_tensor(rp, cl, vl.to(dt), size=(self.n, self.n)).to(device) for dt in (F64, torch.float32)}
        self.T = self                   # A_hat is symmetric: the backward multiplies by A_hat itself
        self._tperm = None

    def dropped_by(self, edge, p):
        """node dropout (the reference's SparseDropout) with the keep bytes `edge` over the CSR slots: a graph whose kept slots
        weigh val * (float)(1 / (1 - p)) in fp32 and whose dropped slots weigh 0, with its transpose as .T (A_drop is not
        symmetric); both as float64 and float32 CSR"""
        kept = torch.as_tensor(edge).to("cpu", torch.bool)
        assert kept.numel() == self.col.numel()
        vl = torch.where(kept, self.val * torch.tensor(np.float32(1.0 / (1.0 - p))), torch.zeros((), dtype=torch.float32))
        if self._tperm is None:          # the slots in (col, row) order: the transpose's CSR order
            rows = torch.repeat_interleave(torch.arange(self.n), self.row_ptr[1:] - self.row_ptr[:-1])
            self._tperm = torch.argsort(self.col * self.n + rows)
            self._trows = rows[self._tperm]
            self._tptr = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(torch.bincount(self.col, minlength=self.n), 0)])
        g = RefGraph(self.row_ptr, self.col, vl, self.device)
        g.T = RefGraph(self._tptr, self._trows, vl[self._tperm], self.device)
        g.T.T = g
        return g

    def dropped(self):
        """the same graph with the last edge of the first multi-segment row removed (a defect of the backward only)"""
        deg = (self.row_ptr[1:] - self.row_ptr[:-1])
        r = int(torch.nonzero(deg > 256)[0])
        e = int(self.row_ptr[r + 1]) - 1
        vl = self.val.clone()
        vl[e] = 0.0
        g = RefGraph.__new__(RefGraph)
        g.n, g.row_ptr, g.col, g.val, g.device = self.n, self.row_ptr, self.col, vl, self.device
        g.A = {dt: torch.sparse_csr_tensor(self.row_ptr, self.col, vl.to(dt), size=(self.n, self.n)).to(self.device)
               for dt in (F64, torch.float32)}
        g.T = g
        g.dropped_row = r
        return g


def spmm(g, X, dt):
    return g.A[dt] @ X


# ---------------------------------------------------------------- shared pieces of the two references
def bpr_head(Rv, RN, RP, U, bu, bi, bj, dt):
    """scores on the representation rows Rv [n, C] (noise RN, discrete RP): -> loss parts and dL/dR (value, N, P)"""
    p, qi, qj = Rv[bu], Rv[U + bi], Rv[U + bj]
    pA, qiA, qjA = _A(p), _A(qi), _A(qj)
    pN, qiN, qjN = RN[bu], RN[U + bi], RN[U + bj]
    pP, qiP, qjP = RP[bu], RP[U + bi], RP[U + bj]
    x = (p * qi).sum(1) - (p * qj).sum(1)
    xN = (pA * (qiA + qjA) + pN * (qiA + qjA) + pA * (qiN + qjN)).sum(1)
    xP = (pP * (qiA + qjA) + pA * (qiP + qjP)).sum(1)
    s = 1.0 / (1.0 + torch.exp(-x))
    c = -(s * (1.0 - s)) / (GAMMA + s)
    lt = -torch.log(GAMMA + s)
    cN = xN / 4 + _A(c)
    cP = xP / 4
    G = torch.zeros(Rv.shape, dtype=dt, device=Rv.device)
    GN = torch.zeros(Rv.shape, dtype=F64, device=Rv.device)
    GP = torch.zeros(Rv.shape, dtype=F64, device=Rv.device)
    d = qi - qj
    cA = _A(c)[:, None]
    G.index_add_(0, bu, c[:, None] * d)
    GN.index_add_(0, bu, cA * (qiA + qjA + qiN + qjN) + cN[:, None] * (qiA + qjA))
    GP.index_add_(0, bu, cA * (qiP + qjP) + cP[:, None] * (qiA + qjA))
    for it, sg in ((U + bi, 1.0), (U + bj, -1.0)):
        G.index_add_(0, it, sg * c[:, None] * p)
        GN.index_add_(0, it, cA * (pA + pN) + cN[:, None] * pA)
        GP.index_add_(0, it, cA * pP + cP[:, None] * pA)
    return dict(loss=float(lt.to(F64).sum()), lossN=float((xN + _A(lt)).sum()), lossP=float(xP.sum())), G, GN, GP



def ego_reg(E0, U, bu, bi, bj, reg, rows_src=None):
    """the regulariser of the ego rows (rows_src: the table the norms and terms are taken on) -> (g, N, loss, lossN)"""
    reg1, reg2 = reg
    src = (E0 if rows_src is None else rows_src).to(F64)
    n = E0.shape[0]
    g = torch.zeros(E0.shape, dtype=F64, device=E0.device)
    N = torch.zeros_like(g)
    lreg = lregN = 0.0
    if not (reg1 or reg2):
        return g, N, 0.0, 0.0
    for idx in (bu, U + bi, U + bj):
        rows = src[idx]
        l1 = float(rows.abs().sum())
        nr = math.sqrt(float((rows ** 2).sum()))
        inv = float(np.float32(1.0 / nr)) if nr > 0 else 0.0
        t = reg1 * torch.sign(rows) + reg2 * rows * inv
        g.index_add_(0, idx, t)
        N.index_add_(0, idx, t.abs())
        lreg += reg1 * l1 + reg2 * nr
        lregN += abs(reg1 * l1) + abs(reg2 * nr)
    return g, N, lreg, lregN


# ---------------------------------------------------------------- LightGCN reference
def lgcn_ref(E0, U, g, L, bu, bi, bj, reg=(0.0, 0.0), dt=F64, defects=()):
    """one LightGCN + BPR step (gradient of E0, not applied) -> dict(g, N, P, loss, lossN, lossP, Em, EmN)"""
    E = E0.to(dt)
    x, xM, xN = E, _A(E0), torch.zeros(E0.shape, dtype=F64, device=E0.device)
    S, SM, SN = E.clone(), xM.clone(), xN.clone()
    for l in range(L):
        x, xN, xM = spmm(g, x, dt), spmm(g, xM + xN, F64), spmm(g, xM, F64)
        if not ("no_last_layer" in defects and l == L - 1):
            S, SM, SN = S + x, SM + xM, SN + xN
    inv = float(np.float32(1.0 / (L + 1)))
    Em = S * inv
    EmN = (SM + SN) * inv + _A(Em)
    head, G, GN, GP = bpr_head(Em, EmN, torch.zeros_like(EmN), U, bu, bi, bj, dt)
    gb = g.dropped() if "drop_edge" in defects else g
    y, yN, yM = G, GN, _A(G)
    T, TN, TM = G.clone(), GN.clone(), yM.clone()
    for l in range(L):
        y, yN, yM = spmm(gb, y, dt), spmm(g, yM + yN, F64), spmm(g, yM, F64)
        T, TN, TM = T + y, TN + yN, TM + yM
    sc = 1.0 if "no_inv" in defects else inv
    gr, grN, lreg, lregN = ego_reg(E0, U, bu, bi, bj, reg, Em if "reg_on_propagated" in defects else None)
    grad = (T * sc).to(F64) + gr
    N = (TM + TN) * sc + grN + _A(grad)
    return dict(g=grad, N=N, P=torch.zeros_like(N), loss=head["loss"] + lreg, lossN=head["lossN"] + lregN + abs(head["loss"] + lreg),
                lossP=0.0, Em=Em, EmN=EmN, flagged=0.0)



# ---------------------------------------------------------------- NGCF reference
def ngcf_layout(dims):
    out, o = [], 0
    for l in range(len(dims) - 1):
        i, p = dims[l], dims[l + 1]
        out.append(dict(W1=(o, o + i * p), b1=(o + i * p, o + i * p + p), W2=(o + i * p + p, o + 2 * i * p + p),
                        b2=(o + 2 * i * p + p, o + 2 * (i * p + p))))
        o += 2 * (i * p + p)
    return out, o


def msg_scale(p):
    """the kernels' message-dropout factor 1.0f / (float)(1 - (double)p) of an fp32 p"""
    return float(np.float32(1.0) / np.float32(1.0 - float(np.float32(p))))


def msg_factors(keep, dims, n, p, dt, device):
    """one forward's message keep bytes (layers concatenated, [n, d_l] each) -> per-layer factors keep * msg_scale(p)"""
    k = torch.as_tensor(keep).to(device)
    out, o = [], 0
    for w in dims[1:]:
        out.append(k[o:o + n * w].view(n, w).to(dt) * msg_scale(p))
        o += n * w
    assert o == k.numel()
    return out


def ngcf_ref(E0, W, U, g, dims, bu, bi, bj, reg=(0.0, 0.0), tower_dtype=0, dt=F64, defects=(), kappa=None, keep=None, p=0.0,
             edge=None, node_p=0.0):
    """one NGCF + BPR step (gradients of E0 and W, not applied) -> dict(gE, NE, PE, gW, NW, PW, loss, lossN, lossP, ALL...).
    keep (message dropout p): the keep bytes of one forward, layers concatenated; edge (node dropout node_p): the keep bytes
    of the CSR slots of g, one mask for every layer.  The masks are given, so they add no P_e term."""
    st = Flags(kappa_of("ngcf", tower_dtype) if kappa is None else kappa)
    ku = st.k * U_RND
    dev = E0.device
    L = len(dims) - 1
    lay, nW = ngcf_layout(dims)
    Wd = W.to(dt)
    bf = tower_dtype == 1
    keep_bf = lambda op, l: bf and not (f"unrounded_{op}" in defects and l == 0)  # a defect: one operand of layer 0 stays fp32
    Z = lambda t: torch.zeros(t.shape, dtype=F64, device=dev)
    mf = None if keep is None else msg_factors(keep, dims, E0.shape[0], p, dt, dev)
    gl = [g] * L                                     # the adjacency of each layer: A_hat, or A_drop (.T: its transpose)
    if edge is not None:
        gl = [g.dropped_by(edge, 0.0 if "node_unscaled" in defects else node_p)] * L   # a defect: kept slots keep val
        if "node_mask_per_layer" in defects:         # a defect: every layer but the first draws its own edge mask
            gl = [gl[0]] + [g.dropped_by(np.random.default_rng(l).random(g.col.numel()) >= node_p, node_p) for l in range(1, L)]
    E, EN, EP = E0.to(dt), Z(E0), Z(E0)
    acts = []
    for l in range(L):
        i, p = dims[l], dims[l + 1]
        W1 = Wd[lay[l]["W1"][0]:lay[l]["W1"][1]].view(p, i)
        W2 = Wd[lay[l]["W2"][0]:lay[l]["W2"][1]].view(p, i)
        b1, b2 = Wd[lay[l]["b1"][0]:lay[l]["b1"][1]], Wd[lay[l]["b2"][0]:lay[l]["b2"][1]]
        X = spmm(gl[l], E, dt)
        XN, XP = spmm(gl[l], _A(E) + EN, F64), spmm(gl[l], EP, F64)
        S, SN, SP = E + X, EN + XN + _A(E + X), EP + XP
        T, TN, TP = X * E, _A(X) * EN + XN * _A(E) + _A(X * E), _A(X) * EP + XP * _A(E)
        Sr, SrN, SrP = rnd(S, SN, SP, st, keep_bf("S", l))
        Tr, TrN, TrP = rnd(T, TN, TP, st, keep_bf("T", l))
        W1r = br(W1) if keep_bf("W1", l) else W1
        W2r = br(W2) if keep_bf("W2", l) else W2
        y1 = mm(Sr, SrN, SrP, W1r, Z(W1r), Z(W1r), True)
        y2 = mm(Tr, TrN, TrP, W2r, Z(W2r), Z(W2r), True)
        y = (y1[0] + b1) + (y2[0] + b2)
        yN = y1[1] + y2[1] + _A(b1) + _A(b2) + _A(y)
        yP = y1[2] + y2[2]
        ey = ku * yN + yP
        unc = y.abs().to(F64) <= ey
        st.add(unc)
        z = torch.where(y > 0, y, 0.2 * y)
        zN, zP = yN, yP
        if mf is not None:                                          # Dropout: one more fp32 product per kept element
            z = z * mf[l]
            zN, zP = zN * _A(mf[l]) + _A(z), zP * _A(mf[l])
        rn = torch.clamp(torch.sqrt((z.to(F64) ** 2).sum(1)), min=1e-12)
        nv = z / rn.to(dt)[:, None]
        nA = _A(nv)
        rnN = (_A(z) * zN).sum(1) / rn                              # noise of ||z||
        En = (zN + nA * (nA * zN).sum(1, keepdim=True)) / rn[:, None] + nA * (rnN / rn)[:, None] + nA
        Ep = (zP + nA * (nA * zP).sum(1, keepdim=True)) / rn[:, None]
        acts.append(dict(E=E, EN=EN, EP=EP, X=X, XN=XN, XP=XP, Sr=Sr, SrN=SrN, SrP=SrP, Tr=Tr, TrN=TrN, TrP=TrP, W1r=W1r, W2r=W2r,
                         W1=W1, W2=W2, y=y, ey=ey, unc=unc, n=nv, nN=En, nP=Ep, rn=rn, rnN=rnN))
        E, EN, EP = nv, En, Ep
    C = sum(dims)
    off = np.concatenate([[0], np.cumsum(dims)]).astype(int)
    ALL = torch.cat([E0.to(dt)] + [a["n"] for a in acts], 1)
    ALLN = torch.cat([Z(E0)] + [a["nN"] for a in acts], 1)
    ALLP = torch.cat([Z(E0)] + [a["nP"] for a in acts], 1)
    head, G, GN, GP = bpr_head(ALL, ALLN, ALLP, U, bu, bi, bj, dt)
    gW, NW, PW = torch.zeros(nW, dtype=F64, device=dev), torch.zeros(nW, dtype=F64, device=dev), torch.zeros(nW, dtype=F64, device=dev)
    dE = dEN = dEP = None
    for l in reversed(range(L)):
        a = acts[l]
        i, p = dims[l], dims[l + 1]
        dn = G[:, off[l + 1]:off[l + 2]]
        dnN, dnP = GN[:, off[l + 1]:off[l + 2]], GP[:, off[l + 1]:off[l + 2]]
        if dE is not None:
            dn, dnN, dnP = dn + dE, dnN + dEN, dnP + dEP
        nv, nA, rn = a["n"], _A(a["n"]), a["rn"][:, None]
        dot = (dn * nv).sum(1, keepdim=True)
        dz = (dn - nv * dot) / rn.to(dt)
        dotN = (_A(dn) * a["nN"] + dnN * nA + _A(dn) * nA).sum(1, keepdim=True)
        dotP = (_A(dn) * a["nP"] + dnP * nA).sum(1, keepdim=True)
        dzN = (dnN + nA * dotN + a["nN"] * _A(dot)) / rn + _A(dz) * (a["rnN"][:, None] / rn + 1)
        dzP = (dnP + nA * dotP + a["nP"] * _A(dot)) / rn
        if mf is not None and "msg_bwd_unmasked" not in defects:   # Dropout backward, on the fp32-rounded dz
            dz = dz * mf[l]
            dzN, dzP = dzN * _A(mf[l]) + _A(dz), dzP * _A(mf[l])
        y = a["y"]
        pos = (y < 0) if "leaky_wrong_side" in defects else (y > 0)
        slope = torch.where(pos, 1.0, 0.2).to(dt)
        dY = dz * slope
        sA = _A(slope)
        unc = a["unc"]
        st.add(unc)
        dYN = torch.where(unc, 0.0, dzN * sA)
        dYP = torch.where(unc, 0.8 * (_A(dz) + ku * dzN + dzP) + dzP * sA, dzP * sA)
        col = dY.to(F64).sum(0)
        colN = (_A(dY) + dYN).sum(0)
        colP = dYP.sum(0)
        for k, nm in enumerate(("b1", "b2")):
            if nm == "b2" and "no_b2_grad" in defects and l == 0:
                continue
            lo, hi = lay[l][nm]
            gW[lo:hi] += col; NW[lo:hi] += colN; PW[lo:hi] += colP
        dYr, dYrN, dYrP = rnd(dY, dYN, dYP, st, keep_bf("dY", l))
        for A_, AN_, AP_, nm in ((a["Sr"], a["SrN"], a["SrP"], "W1"), (a["Tr"], a["TrN"], a["TrP"], "W2")):
            v, N_, P_ = mm(dYr.T.contiguous(), dYrN.T.contiguous(), dYrP.T.contiguous(), A_, AN_, AP_, False)
            lo, hi = lay[l][nm]
            gW[lo:hi] += v.to(F64).reshape(-1); NW[lo:hi] += N_.reshape(-1); PW[lo:hi] += P_.reshape(-1)
        dS = mm(dYr, dYrN, dYrP, a["W1r"], Z(a["W1r"]), Z(a["W1r"]), False)
        dT = mm(dYr, dYrN, dYrP, a["W2r"], Z(a["W2r"]), Z(a["W2r"]), False)
        X, XN, XP, El, ElN, ElP = a["X"], a["XN"], a["XP"], a["E"], a["EN"], a["EP"]
        dEl = dS[0] + dT[0] * X
        dElN = dS[1] + _A(dT[0]) * XN + dT[1] * _A(X) + _A(dT[0] * X) + _A(dEl)
        dElP = dS[2] + _A(dT[0]) * XP + dT[2] * _A(X)
        dX = dS[0] + dT[0] * El
        dXN = dS[1] + _A(dT[0]) * ElN + dT[1] * _A(El) + _A(dT[0] * El) + _A(dX)
        dXP = dS[2] + _A(dT[0]) * ElP + dT[2] * _A(El)
        gt = gl[l] if "node_bwd_untransposed" in defects else gl[l].T    # a defect: A_drop in place of A_drop^T
        AdX, AdXN, AdXP = spmm(gt, dX, dt), spmm(gt, _A(dX) + dXN, F64), spmm(gt, dXP, F64)
        dE, dEN, dEP = dEl + AdX, dElN + AdXN + _A(dEl + AdX), dElP + AdXP
    gE = (dE + G[:, :dims[0]]).to(F64)
    NE = dEN + GN[:, :dims[0]] + _A(gE)
    PE = dEP + GP[:, :dims[0]]
    gr, grN, lreg, lregN = ego_reg(E0, U, bu, bi, bj, reg)
    gE = gE + gr
    NE = NE + grN
    return dict(g=[gE, gW], N=[NE, NW], P=[PE, PW], loss=head["loss"] + lreg,
                lossN=head["lossN"] + lregN + abs(head["loss"] + lreg), lossP=head["lossP"], ALL=ALL, ALLN=ALLN, ALLP=ALLP,
                flagged=st.frac())


def w_sections(dims):
    lay, nW = ngcf_layout(dims)
    return [(f"{k}[{l}]", *lay[l][k]) for l in range(len(lay)) for k in ("W1", "b1", "W2", "b2")]


# ---------------------------------------------------------------- steppers: the device and its CPU stand-in
def lgcn_ws_parts(U, I, F, opt):
    """carve_lgcn (lightgcn.cu): hdr, Em, Xa, Xb, G, Gs, cntU, cntI, [m, v]"""
    tab = 4 * (U + I) * F
    parts = [("hdr", 256), ("Em", tab), ("Xa", tab), ("Xb", tab), ("G", tab), ("Gs", tab), ("cntU", 4 * U), ("cntI", 8 * I)]
    return parts + ([("m", tab), ("v", tab)] if opt == "adam" else [])


def ngcf_ws_parts(U, I, dims, opt):
    """carve_ngcf (ngcf.cu)"""
    n, L, C = U + I, len(dims) - 1, sum(dims)
    nW = ngcf_layout(dims)[1]
    wide = 4 * n * max(dims)
    parts = [("hdr", 256), ("ALL", 4 * n * C), ("G", 4 * n * C)]
    for l in range(L):
        parts += [(f"E{l + 1}", 4 * n * dims[l + 1]), (f"X{l}", 4 * n * dims[l]), (f"Y{l}", 4 * n * dims[l + 1]), (f"rn{l}", 4 * n)]
    parts += [("ST", 2 * wide)] + [(k, wide) for k in ("Y1", "Y2", "dY", "dS", "dT", "dX", "dEa", "dEb", "AdX")]
    parts += [("gE", 4 * n * dims[0]), ("gW", 4 * nW), ("scratch", 64), ("cntU", 4 * U), ("cntI", 8 * I)]
    return parts + ([("mE", 4 * n * dims[0]), ("vE", 4 * n * dims[0]), ("mW", 4 * nW), ("vW", 4 * nW)] if opt == "adam" else [])


class _Graph:
    """LightGCN (dims None) or NGCF on E0 (and W): the reference call and the compared sections"""
    phi_max = PHI_FRAC_MAX

    def _model(self, rg, U, I, L, dims, td):
        self.rg, self.U, self.I, self.L, self.dims, self.td = rg, U, I, L, dims, td
        self.kappa = kappa_of("lgcn" if dims is None else "ngcf", td)
        self.ref_uses_kappa = dims is not None

    def reference(self, pre, idx, kappa, dt=F64, defects=(), keep=None, p=0.0, edge=None, node_p=0.0, forward=None):
        """keep, p, edge, node_p: one step's NGCF dropout masks (ngcf_ref); forward: the step's forward counter (the device's)"""
        if self.dims is None:
            res = lgcn_ref(pre["E0"], self.U, self.rg, self.L, *idx, self.reg, dt, defects)
            return dict(res, g=dict(E0=res["g"]), N=dict(E0=res["N"]), P=dict(E0=res["P"]))
        res = ngcf_ref(pre["E0"], pre["W"], self.U, self.rg, self.dims, *idx, self.reg, self.td, dt, defects, kappa, keep, p, edge,
                       node_p)
        return dict(res, **{x: dict(E0=res[x][0], W=res[x][1]) for x in ("g", "N", "P")})

    def sections(self):
        n, F = self.t["E0"].shape
        return [("E0", "E0", 0, n * F, F)] + ([] if self.dims is None else
                                              [(name, "W", a, b, 1) for name, a, b in w_sections(self.dims)])


class Gpu(_Graph, Stepper):
    """LightGCN or NGCF steps through ops on E0 (and W) held on the GPU"""
    device = "cuda"

    def __init__(self, graph, rg, U, I, E0, W, planes, L, opt, lr, reg, dims=None, tower_dtype=0):
        from daisyrec_b200 import _lib, ops
        self._model(rg, U, I, L, dims, tower_dtype)
        self.ops, self.graph, self.opt, self.lr, self.reg = ops, graph, opt, lr, reg
        self.t = dict(E0=device_tensor(E0).clone().contiguous())
        if W is not None:
            self.t["W"] = device_tensor(W).clone().contiguous()
        self.planes = tuple(device_tensor(p).to(torch.int32).contiguous() for p in planes)
        self.hp = ops.hyper(lr, reg[0], reg[1], opt)
        if dims is None:
            self.ws = ops.LgcnWorkspace(U, I, E0.shape[1], opt, "cuda")
            lay, total = carve(lgcn_ws_parts(U, I, E0.shape[1], opt))
            assert total == _lib.lib().drb_lgcn_workspace_bytes(U, I, E0.shape[1], _lib.OPT_KIND[opt])
            moms = dict(E0=("m", "v"))
        else:
            self.ws = ops.NgcfWorkspace(U, I, dims, opt, "cuda")
            lay, total = carve(ngcf_ws_parts(U, I, dims, opt))
            arr = (__import__("ctypes").c_int32 * len(dims))(*dims)
            assert total == _lib.lib().drb_ngcf_workspace_bytes(U, I, arr, len(dims) - 1, _lib.OPT_KIND[opt])
            moms = dict(E0=("mE", "vE"), W=("mW", "vW"))
        if opt == "adam":
            v = views(self.ws.buf, lay, {k: torch.float32 for mv in moms.values() for k in mv})
            self.mom = {key: (v[m].view(self.t[key].shape), v[s].view(self.t[key].shape)) for key, (m, s) in moms.items()}
        torch.cuda.synchronize()

    def run(self, lo, n, batch, k, adam_step0=0, apply=True, first_step=0, **step):
        assert not step, "steps without dropout (DropGpu of test_gpu_ngcf_dropout_fp64.py takes masks)"
        bu, bi, bj = (p[lo:lo + n] for p in self.planes)
        if self.dims is None:
            out = self.ops.lgcn_bpr_train_steps(self.t["E0"], self.ws, self.graph, self.L, bu, bi, bj, batch, first_step, k,
                                                self.hp, adam_step0=adam_step0, apply=apply)
        else:
            out = self.ops.ngcf_bpr_train_steps(self.t["E0"], self.t["W"], self.ws, self.graph, bu, bi, bj, batch, first_step, k,
                                                self.hp, adam_step0=adam_step0, apply=apply, tower_dtype=self.td)
        torch.cuda.synchronize()
        return out.cpu().numpy()


class StandIn(_Graph, fp64_step.StandIn):
    """CPU stand-in of the device: the reference in float32 (optionally with defects)"""

    def __init__(self, rg, U, I, E0, W, planes, L, opt, lr, reg, dims=None, tower_dtype=0, defects=()):
        super().__init__(dict(E0=E0) if W is None else dict(E0=E0, W=W), planes, opt, lr, reg, defects)
        self._model(rg, U, I, L, dims, tower_dtype)


# ---------------------------------------------------------------- problems
def random_graph(rng, U, I, nnz, zipf=1.15):
    from daisyrec_b200 import ops
    cu = rng.integers(U, size=nnz).astype(np.int32)
    ci = np.minimum(I - 1, rng.zipf(zipf, size=nnz) - 1).astype(np.int32)     # a few items with > 256 neighbours
    return ops.lgcn_norm_adj(cu, ci, U, I)


def crafted_graph(rng):
    """users with degrees 0, 1, 3, 4, 5, 255, 256, 257, 511, 512, 513 and 4 099, then 300 users of degree 2..40"""
    from daisyrec_b200 import ops
    degs = [0, 1, 3, 4, 5, 255, 256, 257, 511, 512, 513, 4099] + list(rng.integers(2, 40, 300))
    U, I = len(degs), 6000
    cu = np.concatenate([np.full(d, u, np.int32) for u, d in enumerate(degs)])
    ci = np.concatenate([rng.choice(I - 1, d, replace=False).astype(np.int32) for d in degs])   # item I - 1: degree 0
    return U, I, ops.lgcn_norm_adj(cu, ci, U, I)


def planes_uniform(rng, U, I, n):
    return (rng.integers(U, size=n).astype(np.int32), rng.integers(I, size=n).astype(np.int32), rng.integers(I, size=n).astype(np.int32))


def amazon_book(B, nsteps, seed=2022):
    """bench shape: device-built adjacency (checked bit-identical to the host build) and bench-style planes"""
    from daisyrec_b200 import ops
    from daisyrec_b200.utils.synthetic import SHAPES, make_interactions
    U, I, nnz = SHAPES["amazon-book"]
    d = make_interactions(U, I, nnz, seed=seed, device="cuda")
    adj = ops.lgcn_build_adj(d["coo_u"], d["coo_i"], U, I)
    host = ops.lgcn_norm_adj(d["coo_u"].cpu().numpy(), d["coo_i"].cpu().numpy(), U, I)
    for a, b in zip(adj, host):
        assert np.array_equal(a.cpu().numpy(), b)
    graph = ops.LgcnGraph(*adj, "cuda")
    rg = RefGraph(*host, "cuda")
    g = torch.Generator(device="cuda"); g.manual_seed(seed + 1)
    idx = torch.randint(0, d["coo_u"].numel(), (nsteps * B,), device="cuda", generator=g)
    planes = (d["coo_u"][idx].contiguous(), d["coo_i"][idx].contiguous(),
              torch.randint(0, I, (nsteps * B,), device="cuda", dtype=torch.int32, generator=g))
    assert np.diff(host[0]).max() > 2000                             # rows of many 256-edge segments
    return U, I, graph, rg, planes, g


@pytest.fixture(scope="module")
def gpu():
    from daisyrec_b200 import ops
    ops.require_cuda()
    return ops


# ---------------------------------------------------------------- GPU: LightGCN
@pytest.mark.gpu
@pytest.mark.parametrize("B", [65536, 1 << 20])
def test_lgcn_bench_trajectory_adam(gpu, B):
    """c4_lightgcn: Amazon-Book shape, F = 64, L = 3, Adam lr 0.01, reg 0; steps 0-2 checked, a stretch in one launch, one more"""
    ns = 8 if B == 65536 else 6
    U, I, graph, rg, planes, g = amazon_book(B, ns)
    E0 = torch.randn(U + I, 64, device="cuda", generator=g) * 0.05
    st = Gpu(graph, rg, U, I, E0, None, planes, 3, "adam", 0.01, (0.0, 0.0))
    recs = [checked_step(st, s * B, B, B, f"adam step {s}", adam_step0=s, ref_device="cuda") for s in range(3)]
    k = ns - 4
    st.run(3 * B, k * B, B, k, adam_step0=3)
    recs.append(checked_step(st, (ns - 1) * B, B, B, f"adam step {ns - 1}", adam_step0=ns - 1, ref_device="cuda"))
    report(f"lgcn bench adam B={B}", recs)


@pytest.mark.gpu
def test_lgcn_bench_shape_sgd_reg(gpu):
    B = 65536
    U, I, graph, rg, planes, g = amazon_book(B, 2, seed=7)
    E0 = torch.randn(U + I, 64, device="cuda", generator=g) * 0.05
    st = Gpu(graph, rg, U, I, E0, None, planes, 3, "sgd", 0.05, (1e-3, 1e-3))
    recs = [checked_step(st, s * B, B, B, f"sgd step {s}", ref_device="cuda") for s in range(2)]
    # nodes more than L hops from every batch row have N = 0 and stayed bit-identical (compare_part's stray count)
    assert all(r["tensors"]["E0"]["stray"] == 0 for r in recs)
    report("lgcn bench sgd reg", recs)


SPMM_F = [1, 2, 3, 4, 6, 8, 16, 33, 65, 128, 130, 256, 512, 1024]


@pytest.mark.gpu
@pytest.mark.parametrize("F", SPMM_F)
def test_spmm_geometry_propagate(gpu, F):
    """drb_lgcn_propagate against fp64 on a graph with degrees 0 .. 4 099 (4-edge loop, tail, one-edge second segments)"""
    ops = gpu
    rng = np.random.default_rng(F)
    U, I, (rp, col, val) = crafted_graph(rng)
    graph = ops.LgcnGraph(rp, col, val, "cuda")
    rg = RefGraph(rp, col, val, "cuda")
    deg = np.diff(rp)
    assert {0, 1, 3, 4, 5, 255, 256, 257, 511, 512, 513, 4099} <= set(deg.tolist())
    E0 = torch.from_numpy((rng.standard_normal((U + I, F)) * 0.3).astype(np.float32)).cuda()
    ws = ops.LgcnWorkspace(U, I, F, "sgd", "cuda")
    worst = 0.0
    for L in (0, 1, 4):
        got = ops.lgcn_propagate(E0, ws, graph, L).to(F64)
        x, xM, xN = E0.to(F64), E0.abs().to(F64), torch.zeros_like(got)
        S, SM, SN = x.clone(), xM.clone(), xN.clone()
        for _ in range(L):
            x, xN, xM = spmm(rg, x, F64), spmm(rg, xM + xN, F64), spmm(rg, xM, F64)
            S, SM, SN = S + x, SM + xM, SN + xN
        want = S / (L + 1)
        bound = KAPPA["lgcn"] * U_RND * (SM + SN) / (L + 1) + 2 * U_RND * want.abs()
        err = (got - want).abs()
        r = float(torch.where(err > 0, err / bound, torch.zeros_like(err)).max())
        worst = max(worst, r)
        assert r <= 1, (F, L, r)
        if L == 0:
            assert torch.equal(got.float(), E0)
    print(f"spmm F={F}: worst error/bound {worst:.3g}")


@pytest.mark.gpu
def test_spmm_unsupported_width_is_an_error(gpu):
    ops = gpu
    rng = np.random.default_rng(1)
    U, I, (rp, col, val) = crafted_graph(rng)
    graph = ops.LgcnGraph(rp, col, val, "cuda")
    E0 = torch.ones(U + I, 257, device="cuda")
    ws = ops.LgcnWorkspace(U, I, 257, "sgd", "cuda")
    with pytest.raises(RuntimeError, match="unsupported factors=257"):
        ops.lgcn_propagate(E0, ws, graph, 1)


def _mid_lgcn(seed, F=64, L=3, opt="sgd", reg=(1e-3, 1e-3), n=6000, lr=0.05, device="cuda"):
    rng = np.random.default_rng(seed)
    U, I = 3000, 2500
    rp, col, val = random_graph(rng, U, I, 40000)
    E0 = (rng.standard_normal((U + I, F)) * 0.1).astype(np.float32)
    planes = planes_uniform(rng, U, I, n)
    return U, I, (rp, col, val), E0, planes, rng


@pytest.mark.gpu
def test_lgcn_launches(gpu):
    """one 5-step launch (first_step 1, short last batch) against five single launches each checked; apply=False; duplicates"""
    ops = gpu
    U, I, adj, E0, planes, rng = _mid_lgcn(3, n=1000 + 4 * 1000 + 1000 + 333)
    rg = RefGraph(*adj, "cuda")
    graph = ops.LgcnGraph(*adj, "cuda")
    B, T = 1000, len(planes[0])
    multi = Gpu(graph, rg, U, I, E0, None, planes, 3, "sgd", 0.05, (1e-3, 1e-3))
    single = Gpu(graph, rg, U, I, E0, None, planes, 3, "sgd", 0.05, (1e-3, 1e-3))
    recs = launch_vs_singles(multi, single, T, B, 5, first_step=2)
    assert recs[4]["nb"] == 333
    # loss only on an Adam workspace after one step: E0 and the moments unchanged
    ad = Gpu(graph, rg, U, I, E0, None, planes, 3, "adam", 0.01, (1e-3, 1e-3))
    recs.append(checked_step(ad, 0, B, B, "adam step 0", ref_device="cuda"))
    recs.append(checked_step(ad, B, B, B, "loss only", adam_step0=1, apply=False, ref_device="cuda"))
    # duplicated triples and i == j
    bu, bi, bj = (p.copy() for p in planes)
    bu[:B // 2], bi[:B // 2], bj[:B // 2] = 7, 11, 13
    bj[B // 2:B] = bi[B // 2:B]
    dup = Gpu(graph, rg, U, I, E0, None, (bu, bi, bj), 3, "sgd", 0.05, (1e-3, 1e-3))
    recs.append(checked_step(dup, 0, B, B, "duplicates and i == j", ref_device="cuda"))
    report("lgcn launches", recs)


# ---------------------------------------------------------------- GPU: NGCF
def ngcf_forward_check(ops, graph, rg, U, I, E0, W, dims, td, keep=None, p=0.0, edge=None, node_p=0.0, got=None):
    """ngcf_forward (or the device forward `got`, e.g. ngcf_forward_philox's) against the reference with the same masks ->
    (worst error/bound at the module's KAPPA, smallest KAPPA of KAPPA_LADDER that bounds every element)"""
    if got is None:
        ws = ops.NgcfWorkspace(U, I, dims, "sgd", "cuda")
        got = ops.ngcf_forward(E0, W, ws, graph, tower_dtype=td, dropout=p, keep=keep)
    got = got.to(F64)
    z = torch.zeros(1, dtype=torch.long, device="cuda")

    def ratio(k):
        res = ngcf_ref(E0, W, U, rg, dims, z, z, z, (0.0, 0.0), td, kappa=k, keep=keep, p=p, edge=edge, node_p=node_p)
        bound = k * U_RND * res["ALLN"] + res["ALLP"] + 2 * U_RND * res["ALL"].abs().to(F64)
        err = (got - res["ALL"].to(F64)).abs()
        return float(torch.where(err > 0, err / bound, torch.zeros_like(err)).max())
    need = next((k for k in KAPPA_LADDER if ratio(k) <= 1), float("inf"))
    return ratio(kappa_of("ngcf", td)), need


@pytest.mark.gpu
@pytest.mark.parametrize("opt,td", [("adam", 0), ("adam", 1), ("sgd", 0), ("sgd", 1)])
def test_ngcf_bench_shape(gpu, opt, td):
    """f_ngcf: Amazon-Book shape, widths 64/64/64/64, B = 65 536; the forward and one checked step, tower_dtype 0 and 1"""
    ops = gpu
    B, dims = 65536, [64, 64, 64, 64]
    U, I, graph, rg, planes, g = amazon_book(B, 2, seed=12)
    E0 = (torch.randn(U + I, 64, device="cuda", generator=g) * 0.05).contiguous()
    W = (torch.randn(ops.ngcf_param_count(dims), device="cuda", generator=g) * 0.1).contiguous()
    r, need = ngcf_forward_check(ops, graph, rg, U, I, E0, W, dims, td)
    print(f"forward td={td}: worst error/bound {r:.3g}, kappa needed {need:.3g}")
    assert r <= 1, r
    lr = 0.001 if opt == "adam" else 0.05
    st = Gpu(graph, rg, U, I, E0, W, planes, 3, opt, lr, (0.0, 1e-3), dims, td)
    recs = [checked_step(st, s * B, B, B, f"{opt} td={td} step {s}", adam_step0=s, ref_device="cuda") for s in range(2)]
    report(f"ngcf bench {opt} td={td}", recs)


NGCF_WIDTHS = [[64, 10], [12, 10, 8], [64, 33, 32], [6, 6], [256, 256], [16, 24, 10, 6, 8]]


@pytest.mark.gpu
@pytest.mark.parametrize("td", [0, 1])
@pytest.mark.parametrize("dims", NGCF_WIDTHS, ids=lambda d: "-".join(map(str, d)))
def test_ngcf_widths(gpu, dims, td):
    ops = gpu
    rng = np.random.default_rng(sum(dims) + td)
    U, I = 1500, 1200
    adj = random_graph(rng, U, I, 20000)
    graph, rg = ops.LgcnGraph(*adj, "cuda"), RefGraph(*adj, "cuda")
    E0 = torch.from_numpy((rng.standard_normal((U + I, dims[0])) * 0.1).astype(np.float32)).cuda()
    W = torch.from_numpy((rng.standard_normal(ops.ngcf_param_count(dims)) * 0.15).astype(np.float32)).cuda()
    r, need = ngcf_forward_check(ops, graph, rg, U, I, E0, W, dims, td)
    print(f"forward {dims} td={td}: worst error/bound {r:.3g}, kappa needed {need:.3g}")
    assert r <= 1, r
    B = 3000
    planes = planes_uniform(rng, U, I, 2 * B)
    st = Gpu(graph, rg, U, I, E0, W, planes, len(dims) - 1, "sgd", 0.05, (1e-3, 1e-3), dims, td)
    recs = [checked_step(st, 0, B, B, f"{dims} td={td} sgd", ref_device="cuda")]
    st = Gpu(graph, rg, U, I, E0, W, planes, len(dims) - 1, "adam", 0.001, (1e-3, 1e-3), dims, td)
    recs += [checked_step(st, s * B, B, B, f"{dims} td={td} adam {s}", adam_step0=s, ref_device="cuda") for s in range(2)]
    report(f"ngcf widths {dims} td={td}", recs)


@pytest.mark.gpu
@pytest.mark.parametrize("td", [0, 1])
def test_ngcf_launches(gpu, td):
    """a 3-step launch (short last batch) against three single launches, each checked, and a loss-only call"""
    ops = gpu
    dims = [32, 32, 16]
    rng = np.random.default_rng(5 + td)
    U, I = 1500, 1200
    adj = random_graph(rng, U, I, 20000)
    graph, rg = ops.LgcnGraph(*adj, "cuda"), RefGraph(*adj, "cuda")
    E0 = (rng.standard_normal((U + I, 32)) * 0.1).astype(np.float32)
    W = (rng.standard_normal(ops.ngcf_param_count(dims)) * 0.15).astype(np.float32)
    B = 2000
    planes = planes_uniform(rng, U, I, 3 * B - 500)
    multi = Gpu(graph, rg, U, I, E0, W, planes, 2, "sgd", 0.05, (1e-3, 1e-3), dims, td)
    single = Gpu(graph, rg, U, I, E0, W, planes, 2, "sgd", 0.05, (1e-3, 1e-3), dims, td)
    recs = launch_vs_singles(multi, single, 3 * B - 500, B, 3)
    recs.append(checked_step(single, 0, B, B, "loss only", apply=False, ref_device="cuda"))
    report(f"ngcf launches td={td}", recs)


# ---------------------------------------------------------------- CPU checks
def _small(seed, F, U=40, I=30, nnz=400, B=97):
    rng = np.random.default_rng(seed)
    cu = rng.integers(U, size=nnz).astype(np.int32)
    ci = np.minimum(I - 1, rng.zipf(1.3, size=nnz) - 1).astype(np.int32)
    from oracle import oracle as orc
    adj = orc.lgcn_norm_adj(cu, ci, U, I)
    return rng, U, I, adj, planes_uniform(rng, U, I, B)


def _oracle_run(orc, model, opt, E0, W, U, I, adj, dims, planes, hp):
    """two oracle steps (step counts 1 and 2) -> [(E, W, m, v, loss)] before step 1, before step 2 and after it; m, v: lists
    per parameter tensor (E0 [, W]) as float64, from the oracle's own Adam state"""
    Eo, Wo = E0.copy(), W.copy()
    nE = E0.size
    if model == "lgcn":
        m, v = np.zeros_like(Eo), np.zeros_like(Eo)
        mv = lambda: ([m.astype(np.float64)], [v.astype(np.float64)])
    else:
        state = np.zeros(2 * (E0.size + W.size), np.float32)
        tot = nE + W.size
        mv = lambda: ([state[:nE].astype(np.float64).reshape(E0.shape), state[nE:tot].astype(np.float64)],
                      [state[tot:tot + nE].astype(np.float64).reshape(E0.shape), state[tot + nE:].astype(np.float64)])
    out = []
    for s, (bu, bi, bj) in enumerate(planes):
        out.append((Eo.copy(), Wo.copy(), *mv()))
        if model == "lgcn":
            lo = orc.lgcn_bpr_step(Eo, U, I, 2, *adj, bu, bi, bj, hp, True, None if opt == "sgd" else (m, v), s + 1)
        else:
            lo = orc.ngcf_bpr_step(Eo, Wo, U, I, np.asarray(dims, np.int32), *adj, bu, bi, bj, hp, True,
                                   None if opt == "sgd" else state, s + 1)
        out[-1] = out[-1] + (lo,)
    out.append((Eo.copy(), Wo.copy(), *mv(), None))
    return out


@pytest.mark.parametrize("model,opt", [("lgcn", "sgd"), ("lgcn", "adam"), ("ngcf", "sgd"), ("ngcf", "adam")])
def test_reference_without_rounding_matches_oracle(orc, model, opt):
    """fp32 tower, float64 reference: two steps of orc.lgcn_bpr_step / orc.ngcf_bpr_step on small problems, regulariser on.
    Each step of the reference starts from the oracle's state before it; under Adam the second step has non-zero moments, so
    the size of the gradient (not only its sign, as in a first step) decides the update"""
    dims = [8, 6, 5]
    F, B = 8, 97
    rng, U, I, adj, (bu, bi, bj) = _small(3 + (model == "ngcf"), F, B=2 * B)
    rg = RefGraph(*adj)
    E0 = (rng.standard_normal((U + I, F)) * 0.3).astype(np.float32)
    W = (rng.standard_normal(orc.ngcf_param_count(dims)) * 0.3).astype(np.float32)
    lr, reg = 0.05, (0.002, 0.003)
    planes = [tuple(np.ascontiguousarray(x[s * B:(s + 1) * B]) for x in (bu, bi, bj)) for s in range(2)]
    traj = _oracle_run(orc, model, opt, E0, W, U, I, adj, dims, planes, orc.hyper(lr, reg[0], reg[1], opt))
    for s in range(2):
        Es, Ws, ms, vs, lo = traj[s]
        idx = [torch.from_numpy(x.astype(np.int64)) for x in planes[s]]
        if model == "lgcn":
            res = lgcn_ref(torch.from_numpy(Es), U, rg, 2, *idx, reg)
            gs, tabs, wants = [res["g"]], [Es], [traj[s + 1][0]]
        else:
            res = ngcf_ref(torch.from_numpy(Es), torch.from_numpy(Ws), U, rg, dims, *idx, reg)
            gs, tabs, wants = res["g"], [Es, Ws], [traj[s + 1][0], traj[s + 1][1]]
        assert abs(res["loss"] - lo) <= 2e-6 * abs(lo), (s, res["loss"], lo)
        for k, (t0, want, g) in enumerate(zip(tabs, wants, gs)):
            th, g = torch.from_numpy(t0).to(F64).reshape(-1), g.reshape(-1)
            if opt == "sgd":
                got = th - lr * g
            else:
                m, v = torch.from_numpy(ms[k]).reshape(-1), torch.from_numpy(vs[k]).reshape(-1)
                got = adam_apply(th, g, m, v, lr, s + 1)
            err = (got - torch.from_numpy(want).to(F64).reshape(-1)).abs()
            # Adam at step 1: elements whose gradient is fp32 noise of zero take a +-lr step of either sign in the oracle
            noise = (g.abs() < 1e-6) if (opt == "adam" and s == 0) else torch.zeros_like(g, dtype=torch.bool)
            assert float(err[~noise].max()) <= 2e-6 * max(1.0, float(np.abs(want).max())), (model, opt, s, k, float(err[~noise].max()))
            if opt == "adam" and s == 1:
                # the check sees the gradient's size: the same update from 1.5 g misses the oracle
                off = (adam_apply(th, 1.5 * g, m, v, lr, 2) - torch.from_numpy(want).to(F64).reshape(-1)).abs()
                assert float(off.max()) > 100 * 2e-6 * max(1.0, float(np.abs(want).max()))


def _cpu_case(model, seed=11, opt="sgd", reg=(1e-3, 1e-3), td=0, dims=(16, 12, 10), L=3, F=16, defects=(), big=False, cls=None):
    """a CPU problem with multi-segment rows; -> (stepper (a StandIn, or cls), graph, B)"""
    rng = np.random.default_rng(seed)
    U, I = (400, 300) if not big else (1200, 900)
    adj = random_graph(rng, U, I, 4000 if not big else 12000, zipf=1.1)
    assert np.diff(adj[0]).max() > 256
    rg = RefGraph(*adj)
    Fm = F if model == "lgcn" else dims[0]
    E0 = (rng.standard_normal((U + I, Fm)) * 0.2).astype(np.float32)
    W = None if model == "lgcn" else (rng.standard_normal(ngcf_layout(list(dims))[1]) * 0.2).astype(np.float32)
    B = 700
    planes = planes_uniform(rng, U, I, 2 * B)
    lr = 0.05 if opt == "sgd" else 0.01
    st = (cls or StandIn)(rg, U, I, E0, W, planes, L if model == "lgcn" else len(dims) - 1, opt, lr, reg,
                          None if model == "lgcn" else list(dims), td, defects)
    return st, rg, B


@pytest.mark.parametrize("model,opt,td", [("lgcn", "sgd", 0), ("lgcn", "adam", 0), ("ngcf", "sgd", 0), ("ngcf", "adam", 0),
                                          ("ngcf", "sgd", 1), ("ngcf", "adam", 1)])
def test_harness_passes_with_fp32_stand_in(model, opt, td):
    st, rg, B = _cpu_case(model, opt=opt, td=td, reg=(0.0, 0.0) if opt == "adam" else (1e-3, 1e-3))
    for s in range(2):
        r = checked_step(st, s * B, B, B, f"stand-in {model} {opt} td={td} {s}", adam_step0=s)
        assert r["ok"], summary(r)


DEFECTS = {
    # defect: (model, optimiser, reg, tower_dtype, tensors that must exceed the bound)
    "drop_edge": ("lgcn", "sgd", (1e-3, 1e-3), 0, {"E0"}),
    "no_inv": ("lgcn", "adam", (0.0, 0.0), 0, {"E0"}),
    "no_last_layer": ("lgcn", "sgd", (1e-3, 1e-3), 0, {"E0"}),
    "reg_on_propagated": ("lgcn", "sgd", (1e-2, 1e-2), 0, {"E0"}),
    "no_b2_grad": ("ngcf", "sgd", (1e-3, 1e-3), 0, {"b2[0]"}),
    "leaky_wrong_side": ("ngcf", "sgd", (1e-3, 1e-3), 0, {"E0", "W1[0]", "W2[0]", "b1[0]", "b2[0]"}),
    "unrounded_S": ("ngcf", "sgd", (1e-3, 1e-3), 1, {"E0", "W1[0]"}),
    "unrounded_T": ("ngcf", "sgd", (1e-3, 1e-3), 1, {"E0", "W2[0]"}),
    "unrounded_W1": ("ngcf", "sgd", (1e-3, 1e-3), 1, {"E0"}),
    "unrounded_W2": ("ngcf", "sgd", (1e-3, 1e-3), 1, {"E0"}),
    "unrounded_dY": ("ngcf", "sgd", (1e-3, 1e-3), 1, {"E0", "W1[0]", "W2[0]"}),
}


@pytest.mark.parametrize("defect", sorted(DEFECTS))
def test_harness_flags_defective_stand_in(defect):
    model, opt, reg, td, want = DEFECTS[defect]
    st, rg, B = _cpu_case(model, opt=opt, reg=reg, td=td, defects=(defect,))
    r = checked_step(st, 0, B, B, defect)
    assert not r["ok"], summary(r)
    bad = {k for k, v in r["tensors"].items() if v["ratio"] > 1 or v["unflagged"] > 0}
    assert bad & want, (defect, bad)
    st, rg, B = _cpu_case(model, opt=opt, reg=reg, td=td)
    ok = checked_step(st, 0, B, B, "no defect")
    assert ok["ok"], summary(ok)


def test_staging_predicate_never_loads_misaligned():
    """umma_stage_tile's 16-byte path, mirrored over every NGCF and NeuMF layer-wise call site: the predicate with the base
    check never issues a misaligned load; the one before it did for the widths that motivated the check"""
    bad_before = [[64, 10], [64, 6, 6], [64, 33, 32], [10, 10], [12, 10, 8]]
    fine_before = [[64, 64, 64, 64], [64, 32, 16], [32, 100, 100]]
    for dims in bad_before + fine_before + NGCF_WIDTHS + [[256, 256, 256]]:
        ops_ = ngcf_gemm_operands(dims, ws_base=1 << 20, w_base=1 << 24)
        for site, base, ld, mn, rows, K in ops_:
            assert all(a % 16 == 0 for a in stage_vec_loads(base, ld, mn, rows, K)), (dims, site)
        before = [site for site, base, ld, mn, rows, K in ops_ if any(a % 16 for a in stage_vec_loads(base, ld, mn, rows, K, False))]
        if dims in bad_before:
            assert before, dims
        if dims in fine_before:
            assert not before, (dims, before)
    for F, L in [(4, 1), (12, 2), (24, 2), (32, 2), (64, 1), (64, 3), (128, 2), (128, 3)]:
        for site, base, ld, mn, rows, K in neumf_gemm_operands(F, L, ws_base=1 << 20, w_base=1 << 24):
            v = stage_vec_loads(base, ld, mn, rows, K)
            assert v == stage_vec_loads(base, ld, mn, rows, K, False), (F, L, site)   # aligned: the same vector loads as before
    # the bench widths keep the vector path on every operand
    for site, base, ld, mn, rows, K in ngcf_gemm_operands([64, 64, 64, 64], ws_base=1 << 20, w_base=1 << 24):
        assert stage_vec_loads(base, ld, mn, rows, K) == stage_vec_loads(base, ld, mn, rows, K, False) != [], site
