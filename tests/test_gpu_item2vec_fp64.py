"""Item2Vec: teacher-forced steps of drb_i2v_train_steps and the user-embedding build of drb_i2v_user_embedding against
float64 references, on the shared harness (fp64_step.py).

The step is the point-wise CL branch of the GEN instantiation of the step kernel (step_kernel.cuh) run with U = 0: one tied
table, P == Q and gP == gQ, the first operand counted in cntI, a dense phase-2 sweep.  `i2v_ref` runs it on a snapshot of the
table (and the optimiser state, read from the workspace through a mirror of carve with U = 0): x = Q[t] . Q[c] in float64;
the loss (1 - y) x - log_sigmoid(x) and its coefficient c = (1 - y) - sigmoid(-x); both contributions land in the one table,
g[t] += c Q[c] and g[c] += c Q[t] (a row with t == c takes 2 c Q[t]).  The noise scale N of an element is the sum of
|contributions| to it, each carrying the coefficient's noise (the dot product's sum of |products| through sigmoid' <= 1/4, plus
the fp32 rounding of expf / log1pf); the loss bound adds the per-warp fp32 partials (at most 64 triples of a 512-row tile, then
a 32-lane butterfly) that are widened to float64 in shared memory.  fp32 throughout and no gate: P = 0.  The reference reads
only the pre-step snapshot and the pre-step moments, and runs in blocks of ROW_BLOCK rows, so a B = 2^20 step stays within a
few GB.

Cases: a geometry sweep over every (VEC, W, NCH) lane geometry the GEN kernel dispatches and both sides of its W >= UNR branch
(F in SWEEP_F, I = 2 003) at B = 1, 17 and 4 099 under SGD and Adam (adam_step0 = 0, 1 and 10^4), with t == c rows, an item in
every row of a batch and labels -1 and 2; F = 257 and 1 028 refused before any launch; the ML-20M skip-gram shape (the rows of
scripts/bench_item2vec.py, window 2, permuted on the device) at F = 100: three Adam steps at B = 2^20 and at B = 256, one SGD
step at B = 2^20, a 4-step SGD launch with a ragged last batch against four single launches, one loss-only call after an Adam
step, one Adam step repeated from the same snapshot; the user embedding, bit for bit against a sequential fp32 sum in CSR
order and within (n - 1) u sum|Q| of the float64 sum, at F = 1, 31, 32, 33, 100, 1 024 and at the ML-20M shape; one
Item2Vec.fit epoch (64 Ki rows less 100, B = 256) under Adam and under SGD against single checked steps over the loader's
order.

Calibrated on one H100 80GB HBM3 (700 W power limit).  "Needed" is the per-element KAPPA of an SGD step, else (Adam) the
smallest KAPPA of KAPPA_LADDER at which every element of the step passes.
- geometry sweep: needed 1.14 under SGD (F = 32; <= 0.61 at every other F), 0.5 under Adam;
- bench shape: needed 1.67 for the first SGD step at B = 2^20 (hottest row about 8 950 contributions per step), 3.9 - 4.1 for
  the second step of the 4-step SGD launch, where the tables have grown (<= 2.5 for its other steps), 1 under Adam at B = 2^20,
  0.125 at B = 256;
- fit epoch: needed 0.80 (SGD) and 1 (Adam) over the 256 single steps;
hence KAPPA = 8, twice the largest.  At KAPPA = 8 the worst error / bound is 0.50 in the sweep, 0.49 at the bench
shape and 0.50 over the fit epoch's single steps; the fit's SGD table uses at most 0.0066 of the launch bound.  The
repeated B = 2^20 Adam step gives bitwise equal losses, but about 45 000 elements of Q differ (by up to 7.8e-7), as do the
moments: the gradient sums are fp32 atomics, so that is reported, not asserted.  The user embedding is bitwise equal to the
sequential fp32 sum in every case; its error against the float64 sum reaches 0.9995 of (n - 1) u sum|Q| (two-item rows,
where that bound is tight) and 0.51 at the ML-20M shape, whose longest user row has 2 258 items (a crafted 12 000-item user is
appended).  The new GPU cases take 25 s there, the 1.3 - 3.4 s build of the 158 M skip-gram rows included.  The CPU part
runs the same checks with the reference in float32 standing in for the device on the sweep's small cases, and shows that each
of these defects fails them: a t == c row adding its contribution once, one contribution to the hottest row dropped, the last
row of a ragged batch skipped, Adam's bias correction taken at step t - 1, one row's label read as 1 - y.
"""
import functools
import os
import sys
import time
from types import SimpleNamespace

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fp64_step  # noqa: E402
from fp64_step import (F64, U_RND, Stepper, _A, carve, checked_step, device_tensor, launch_vs_singles,  # noqa: E402
                       report, summary, views)

KAPPA = 8.0
ROW_BLOCK = 1 << 17       # batch rows the reference holds at once
LOSS_PARTIAL = 64 + 5     # terms of the longest fp32 partial sum of the loss: 512-row tile / 8 warps, then 5 butterfly levels

# ---------------------------------------------------------------- the GEN kernel's lane geometry
# mirrors row_geom (common.cuh), the GEN instantiations of pick_kernel_v (mf_bpr.cu) and UNR of bpr_steps_body (step_kernel.cuh)
DISPATCHED = {(1, 1), (2, 1), (4, 1), (8, 1), (16, 1), (32, 1), (32, 2), (32, 4), (32, 8)}


def row_geom(F):
    vec = 4 if F % 4 == 0 else 2 if F % 2 == 0 else 1
    chunks = F // vec
    w = 1
    while w < chunks and w < 32:
        w <<= 1
    per = -(-chunks // w)
    nch = 1
    while nch < per:
        nch <<= 1
    return vec, w, nch


def unr(vec, nch):
    return 2 if nch * vec <= 4 else 1


def supported(F):
    return F > 0 and row_geom(F)[1:] in DISPATCHED


SWEEP_F = (1, 2, 3, 4, 6, 8, 30, 32, 66, 100, 129, 200, 255, 512, 1024)
SWEEP_I = 2003
SWEEP_B = (1, 17, 4099)
ADAM_STEP0 = (0, 1, 10 ** 4)
HOT = 5                   # the item in every row of a B = 17 batch, and in every row but the t == c ones of a B = 4 099 batch


# ---------------------------------------------------------------- workspace mirror
def i2v_ws_layout(I, F, opt):
    """mirror of carve (step.cuh) with U = 0: the user parts take no bytes"""
    parts = [("hdr", 256), ("gP", 0), ("gQ", 4 * I * F), ("cntU", 0), ("cntI", 8 * I)]
    if opt == "adam":
        parts += [("mP", 0), ("vP", 0), ("mQ", 4 * I * F), ("vQ", 4 * I * F)]
    return carve(parts)


# ---------------------------------------------------------------- float64 reference
def i2v_ref(Q, t, c, y, dt=F64, defects=()):
    """one skip-gram step on the tied table Q (gradients, not applied) -> dict(g, N, P: {"Q"}, loss, lossN, lossP, flagged,
    hot: the largest number of contributions one row receives)"""
    I, F = Q.shape
    dev = Q.device
    Qd = Q.to(dt)
    g, N = torch.zeros(I, F, dtype=F64, device=dev), torch.zeros(I, F, dtype=F64, device=dev)
    B = t.numel()
    cnt = torch.bincount(t, minlength=I) + torch.bincount(c, minlength=I)
    keep_t = torch.ones(B, dtype=torch.bool, device=dev)
    keep_c = keep_t.clone()
    if "tc_once" in defects:                       # a t == c row adds its contribution once
        keep_c &= t != c
    if "drop_hot" in defects:                      # the first contribution to the hottest row is lost
        keep_t[int(torch.nonzero(t == int(cnt.argmax()))[0])] = False
    loss = lossN = 0.0
    for a in range(0, B, ROW_BLOCK):
        b = min(B, a + ROW_BLOCK)
        tt, cc, yy = t[a:b], c[a:b], y[a:b].to(dt)
        qt, qc = Qd[tt], Qd[cc]
        x = (qt * qc).sum(1)
        xN = (_A(qt) * _A(qc)).sum(1) + _A(x)
        z = torch.exp(-x.abs())
        dls = torch.where(x < 0, 1 - z / (1 + z), z / (1 + z))       # sigmoid(-x)
        coef = (1 - yy) - dls
        logsig = torch.clamp(x, max=0) - torch.log1p(z)
        lt = (1 - yy) * x - logsig
        cN = xN / 4 + _A(1 - yy) + _A(dls) + _A(coef)
        gt, gc = coef[:, None] * qc, coef[:, None] * qt
        kt, kc = keep_t[a:b], keep_c[a:b]
        g.index_add_(0, tt[kt], gt[kt].to(F64))
        N.index_add_(0, tt[kt], (cN[:, None] * _A(qc) + _A(gt))[kt])
        g.index_add_(0, cc[kc], gc[kc].to(F64))
        N.index_add_(0, cc[kc], (cN[:, None] * _A(qt) + _A(gc))[kc])
        loss += float(lt.to(F64).sum())
        lossN += float((_A(coef) * xN + _A((1 - yy) * x) + _A(logsig) + LOSS_PARTIAL * _A(lt)).sum())
    N += _A(g)
    return dict(g=dict(Q=g), N=dict(Q=N), P=dict(Q=torch.zeros_like(N)), loss=loss, lossN=lossN + abs(loss), lossP=0.0,
                flagged=0.0, hot=int(cnt.max()) if B else 0)


# ---------------------------------------------------------------- steppers: the device and its CPU stand-in
class _Model:
    phi_max = 0.0
    ref_uses_kappa = False            # N does not depend on KAPPA: the ladder reuses one reference result
    reg = 0.0

    def _model(self, I, F):
        self.I, self.F, self.kappa = I, F, KAPPA

    def reference(self, pre, idx, kappa, dt=F64, defects=()):
        return i2v_ref(pre["Q"], *idx, dt, defects)

    def sections(self):
        return [("Q", "Q", 0, self.I * self.F, self.F)]

    def checks(self, pre, post, res, apply):
        return dict(clean=self.clean())


class I2vGpu(_Model, Stepper):
    device = "cuda"

    def __init__(self, Q, planes, opt, lr):
        from daisyrec_b200 import _lib, ops
        self.ops, self.opt, self.lr = ops, opt, lr
        self.Q = device_tensor(Q).float().clone().contiguous()
        self.t = dict(Q=self.Q)
        self._model(*self.Q.shape)
        self.planes = tuple(device_tensor(p).to(torch.int32).contiguous() for p in planes)
        self.hp = ops.hyper(lr, 0.0, 0.0, opt, loss="CL")
        self.ws = ops.I2VWorkspace(self.I, self.F, opt, "cuda")
        lay, total = i2v_ws_layout(self.I, self.F, opt)
        assert total == _lib.lib().drb_i2v_workspace_bytes(self.I, self.F, _lib.OPT_KIND[opt])
        self.acc = views(self.ws.buf, lay, dict(gQ=torch.float32, cntI=torch.int64))
        if opt == "adam":
            v = views(self.ws.buf, lay, dict(mQ=torch.float32, vQ=torch.float32))
            self.mom = {"Q": (v["mQ"], v["vQ"])}
        torch.cuda.synchronize()

    def run(self, lo, n, batch, k, adam_step0=0, apply=True, first_step=0):
        bt, bc, bl = (p[lo:lo + n] for p in self.planes)
        out = self.ops.i2v_train_steps(self.Q, self.ws, bt, bc, bl, batch, first_step, k, self.hp, adam_step0=adam_step0,
                                       apply=apply)
        torch.cuda.synchronize()
        return out.cpu().numpy()

    def clean(self):
        torch.cuda.synchronize()
        return all(int(torch.count_nonzero(v)) == 0 for v in self.acc.values())


class StandIn(_Model, fp64_step.StandIn):
    """CPU stand-in of the device: the reference in float32, optionally with a defect"""

    def __init__(self, Q, planes, opt, lr, defects=()):
        super().__init__(dict(Q=Q), planes, opt, lr, 0.0, defects)
        self._model(*self.t["Q"].shape)

    def stand_in_ref(self, idx):
        if "skip_last_row" in self.defects:
            idx = tuple(x[:-1] for x in idx)
        if "label_flip" in self.defects:            # row 0's label read as 1 - y
            y = idx[2].clone()
            y[0] = 1 - y[0]
            idx = (idx[0], idx[1], y)
        return self.reference(self.t, idx, self.kappa, torch.float32, self.defects)

    def run(self, lo, n, batch, k, adam_step0=0, apply=True, first_step=0):
        if "adam_bc_prev" in self.defects:          # Adam's bias correction taken at step t - 1
            adam_step0 -= 1
        return super().run(lo, n, batch, k, adam_step0, apply, first_step)


# ---------------------------------------------------------------- problems
def sweep_batch(rng, I, nb, kind):
    """one batch of (target, context, label) rows: labels in {-1, 0, 1, 2}; kind "hot": HOT in every row, rows 0, 5, 10, ..
    are (HOT, HOT); kind "mixed": HOT in every row but rows 3, 10, 17, .., which are t == c on random items"""
    t, c = rng.integers(0, I, nb), rng.integers(0, I, nb)
    y = rng.choice(np.array([0, 1, 0, 1, 2, -1]), nb)
    k = np.arange(nb)
    t[k % 2 == 0] = HOT
    c[k % 2 == 1] = HOT
    if kind == "hot":
        t[k % 5 == 0] = c[k % 5 == 0] = HOT
    else:
        tc = k % 7 == 3
        t[tc] = c[tc] = rng.integers(HOT + 1, I, int(tc.sum()))
    return np.stack([t, c, y])


def sweep_plan(opt):
    """[(B, adam_step0)] of one sweep case, in step order"""
    if opt == "sgd":
        return [(B, 0) for B in SWEEP_B]
    return [(B, s0) for s0 in ADAM_STEP0 for B in SWEEP_B]


def sweep_problem(F, opt, seed=0):
    rng = np.random.default_rng(1000 * F + (opt == "adam") + seed)
    Q = (rng.standard_normal((SWEEP_I, F)) * 0.3).astype(np.float32)
    plan = sweep_plan(opt)
    planes = np.concatenate([sweep_batch(rng, SWEEP_I, B, "hot" if B == 17 else "mixed") for B, _ in plan], 1)
    lr = 0.01 if opt == "sgd" else 0.005
    return Q, planes, plan, lr


def run_plan(st, plan, tag, ref_device):
    recs, lo = [], 0
    for B, s0 in plan:
        recs.append(checked_step(st, lo, B, B, f"{tag} B={B} t0={s0}", adam_step0=s0, ref_device=ref_device))
        lo += B
    return recs


# ---------------------------------------------------------------- CPU checks
def test_sweep_table_covers_every_geometry():
    geo = {F: row_geom(F) for F in SWEEP_F}
    assert all(supported(F) for F in SWEEP_F)
    assert {(w, n) for _, w, n in geo.values()} == DISPATCHED                          # every dispatched (W, NCH)
    sides = {(v, w >= unr(v, n)) for v, w, n in geo.values()}
    assert sides == {(v, s) for v in (1, 2, 4) for s in (False, True)}                 # each VEC on both sides of W >= UNR
    assert {unr(v, n) for v, w, n in geo.values()} == {1, 2}
    assert 1024 in SWEEP_F and 255 in SWEEP_F
    assert max(F for F in range(1, 1025) if F % 2 and supported(F)) == 255             # the largest odd supported F
    assert max(F for F in range(1, 2049) if supported(F)) == 1024
    assert not supported(257) and not supported(1028)
    # the table as written: removing any F whose (VEC, W, NCH) no other F has fails the two coverage checks above
    assert set(geo.values()) == {(1, 1, 1), (2, 1, 1), (1, 4, 1), (4, 1, 1), (2, 4, 1), (4, 2, 1), (2, 16, 1), (4, 8, 1),
                                 (2, 32, 2), (4, 32, 1), (1, 32, 8), (4, 32, 2), (4, 32, 4), (4, 32, 8)}


def test_workspace_mirror_matches_library():
    from daisyrec_b200 import _lib
    lib = _lib.lib()
    for I, F in [(1, 1), (3, 7), (2003, 100), (2003, 255), (26744, 100), (26744, 1024)]:
        for opt in ("sgd", "adam"):
            assert i2v_ws_layout(I, F, opt)[1] == lib.drb_i2v_workspace_bytes(I, F, _lib.OPT_KIND[opt])


def test_sweep_batches_hold_the_stress_rows():
    rng = np.random.default_rng(0)
    t, c, y = sweep_batch(rng, SWEEP_I, 17, "hot")
    k5 = np.arange(17) % 5 == 0
    assert ((t == HOT) | (c == HOT)).all() and (t[k5] == HOT).all() and (c[k5] == HOT).all()
    t, c, y = sweep_batch(rng, SWEEP_I, 4099, "mixed")
    tc = np.arange(4099) % 7 == 3
    assert (t[tc] == c[tc]).all() and (t[tc] != HOT).all() and ((t == HOT) | (c == HOT))[~tc].all()
    assert {-1, 2} <= set(y.tolist())


CPU_F = (1, 2, 4, 6, 30, 100, 129)


@pytest.mark.parametrize("opt", ["sgd", "adam"])
@pytest.mark.parametrize("F", CPU_F)
def test_rehearsal_on_stand_in(F, opt):
    Q, planes, plan, lr = sweep_problem(F, opt)
    st = StandIn(Q, planes, opt, lr)
    for r in run_plan(st, plan, f"stand-in F={F} {opt}", "cpu"):
        assert r["ok"], summary(r)


DEFECTS = {
    # defect: (optimiser, F, adam_step0 of the checked step)
    "tc_once": ("sgd", 30, 0),
    "drop_hot": ("sgd", 100, 0),
    "skip_last_row": ("sgd", 6, 0),
    "adam_bc_prev": ("adam", 8, 1),
    "label_flip": ("sgd", 129, 0),
}


@pytest.mark.parametrize("defect", sorted(DEFECTS))
def test_rehearsal_flags_defective_stand_in(defect):
    """each defect fails the check of a B = 4 099 step, run as the ragged last batch of a 5 000-row batch size"""
    opt, F, s0 = DEFECTS[defect]
    rng = np.random.default_rng(7)
    Q = (rng.standard_normal((SWEEP_I, F)) * 0.3).astype(np.float32)
    planes = np.concatenate([sweep_batch(rng, SWEEP_I, 5000, "mixed"), sweep_batch(rng, SWEEP_I, 4099, "mixed")], 1)
    lr = 0.01 if opt == "sgd" else 0.005
    good = StandIn(Q, planes, opt, lr)
    bad = StandIn(Q, planes, opt, lr, defects=(defect,))
    ok = checked_step(good, 5000, 4099, 5000, f"{defect} (correct)", adam_step0=s0)
    r = checked_step(bad, 5000, 4099, 5000, defect, adam_step0=s0)
    print(f"{defect}: ok={r['ok']} worst ratio {r['ratio']:.3g} loss ratio {r['loss_ratio']:.3g} "
          f"stray={sum(c.get('stray', 0) for c in r['tensors'].values())}")
    assert ok["ok"], summary(ok)
    assert not r["ok"], summary(r)


def test_user_sum_reference_order():
    """seq_sum_fp32 adds in CSR order: a row (2^24, 1, -2^24) sums to 0, its reverse to 1"""
    Q = torch.tensor([[2.0 ** 24], [1.0], [-(2.0 ** 24)]])
    row_ptr, col = torch.tensor([0, 3, 6, 6]), torch.tensor([0, 1, 2, 2, 1, 0], dtype=torch.int32)
    P = torch.full((3, 1), 7.0)
    got = seq_sum_fp32(Q, row_ptr, col, P)
    assert got[:, 0].tolist() == [0.0, 1.0, 7.0]


# ---------------------------------------------------------------- user embedding references
def seq_sum_fp32(Q, row_ptr, col, P):
    """P with P[u] = the fp32 sum of Q over the user's CSR row, added one item at a time in col order (round to nearest after
    every addition, no FMA), for the users with a non-empty row; on Q's device"""
    dev = Q.device
    row_ptr, col = row_ptr.to(dev), col.to(dev).long()
    out = P.to(dev).clone()
    length = row_ptr[1:] - row_ptr[:-1]
    order = torch.argsort(length, descending=True, stable=True)
    ls = length[order]
    start = row_ptr[:-1][order]
    neg = -ls.cpu().numpy()
    act = int(np.searchsorted(neg, 0))                        # users with a non-empty row: a prefix of the order
    s = torch.zeros(act, Q.shape[1], dtype=torch.float32, device=dev)
    for k in range(-int(neg[0]) if act else 0):
        na = int(np.searchsorted(neg, -k))                    # users with more than k items
        s[:na] += Q[col[start[:na] + k]]
    out[order[:act]] = s
    return out


def sum_fp64(Q, row_ptr, col):
    """(float64 sums, sums of |Q|, n) of every user's row"""
    dev = Q.device
    row_ptr, col = row_ptr.to(dev), col.to(dev).long()
    n = row_ptr[1:] - row_ptr[:-1]
    u = torch.repeat_interleave(torch.arange(n.numel(), device=dev), n)
    Qd = Q.to(F64)
    s, a = (torch.zeros(n.numel(), Q.shape[1], dtype=F64, device=dev) for _ in range(2))
    s.index_add_(0, u, Qd[col]); a.index_add_(0, u, Qd[col].abs())
    return s, a, n


def check_user_embedding(Q, row_ptr, col, P0, tag):
    """drb_i2v_user_embedding against the sequential fp32 sum (bitwise) and the float64 sum -> record"""
    from daisyrec_b200 import ops
    P = P0.clone()
    ops.i2v_user_embedding(Q, row_ptr, col, P)
    want = seq_sum_fp32(Q, row_ptr, col, P0)
    s, a, n = sum_fp64(Q, row_ptr, col)
    empty = n == 0
    err = (P.to(F64) - s).abs()[~empty]
    bound = (n[~empty] - 1).to(F64)[:, None] * U_RND * a[~empty]
    ratio = float(torch.where(err > 0, err / bound, torch.zeros_like(err)).max())
    rec = dict(tag=tag, bitwise=bool(torch.equal(P, want)), fp64_ratio=ratio, empty_kept=bool(torch.equal(P[empty], P0[empty])),
               users=int(n.numel()), longest=int(n.max()), empty=int(empty.sum()))
    rec["ok"] = rec["bitwise"] and ratio <= 1 and rec["empty_kept"]
    print(f"  {tag}: users {rec['users']} (empty {rec['empty']}), longest row {rec['longest']}, bitwise {rec['bitwise']}, "
          f"fp64 error/bound {ratio:.3g}, empty rows kept {rec['empty_kept']}")
    return rec


def resident_warps():
    """warps of the user-sum launch: grid_for(U * 32, 256) caps the grid at 16 CTAs of 8 warps per SM"""
    return torch.cuda.get_device_properties(0).multi_processor_count * 16 * 8


# ---------------------------------------------------------------- GPU: geometry sweep
@pytest.fixture(scope="module")
def gpu():
    from daisyrec_b200 import ops
    ops.require_cuda()
    return ops


@pytest.mark.gpu
@pytest.mark.parametrize("opt", ["sgd", "adam"])
@pytest.mark.parametrize("F", SWEEP_F)
def test_sweep(gpu, F, opt):
    t0 = time.perf_counter()
    Q, planes, plan, lr = sweep_problem(F, opt)
    st = I2vGpu(Q, planes, opt, lr)
    v, w, n = row_geom(F)
    recs = run_plan(st, plan, f"F={F} {opt}", "cuda")
    report(f"i2v sweep F={F} (VEC {v}, W {w}, NCH {n}, UNR {unr(v, n)}) {opt}", recs)
    print(f"[i2v sweep F={F} {opt}] {time.perf_counter() - t0:.1f} s")


@pytest.mark.gpu
@pytest.mark.parametrize("F", [257, 1028])
def test_unsupported_factors_refused(gpu, F):
    from daisyrec_b200._lib import DrbError
    Q = torch.randn(50, F, device="cuda")
    Q0 = Q.clone()
    ws = gpu.I2VWorkspace(50, F, "adam", Q.device)
    planes = [torch.zeros(8, dtype=torch.int32, device="cuda") for _ in range(3)]
    with pytest.raises(DrbError, match="unsupported factors"):
        gpu.i2v_train_steps(Q, ws, *planes, 8, 0, 1, gpu.hyper(0.01, 0.0, 0.0, "adam", loss="CL"))
    torch.cuda.synchronize()
    assert torch.equal(Q, Q0) and int(torch.count_nonzero(ws.buf)) == 0        # nothing ran


# ---------------------------------------------------------------- GPU: the ML-20M skip-gram shape
ML20M = (138493, 26744, 20_000_263)
BENCH_F = 100
BENCH_ROWS = 8 << 20      # permuted rows kept for the cases below


@functools.lru_cache(maxsize=1)
def _bench():
    """the skip-gram rows of scripts/bench_item2vec.py (window 2, numpy's MT19937 seeded 2022) at the ML-20M shape, permuted on
    the device with a fixed seed so that batches mix users as fit's shuffle does; the first BENCH_ROWS of them"""
    from daisyrec_b200 import ops
    from daisyrec_b200.utils import synthetic
    t0 = time.perf_counter()
    U, I, nnz = ML20M
    d = synthetic.make_interactions(U, I, nnz, device="cuda")
    seq_ptr, ctx_ptr, order = ops.skipgram_group(d["coo_u"], U, 2)
    total = int(ctx_ptr[-1].item())
    draws = ops.skipgram_draws_mt19937(ops.mt19937_seed(2022), I - np.diff(d["row_ptr"].cpu().numpy()),
                                       np.diff(seq_ptr.cpu().numpy()), 2, total)
    rows = ops.skipgram_emit(d["coo_u"], d["coo_i"], order, 2, seq_ptr, ctx_ptr, d["row_ptr"], d["col"],
                             torch.from_numpy(draws).cuda(), total)
    g = torch.Generator(device="cuda")
    g.manual_seed(2023)
    perm = torch.randperm(rows.shape[0], generator=g, device="cuda")[:BENCH_ROWS]
    sub = rows[perm]
    out = SimpleNamespace(U=U, I=I, n_rows=int(rows.shape[0]), planes=tuple(sub[:, k].contiguous() for k in range(3)),
                          rows=sub, row_ptr=d["row_ptr"], col=d["col"])
    del rows, perm, draws
    torch.cuda.empty_cache()
    print(f"[i2v bench shape] {out.n_rows} skip-gram rows, {time.perf_counter() - t0:.1f} s to build")
    return out


def _bench_q(seed, std=0.1):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    return torch.randn(ML20M[1], BENCH_F, generator=g, device="cuda") * std


def _hot(res):
    return f"hottest row {res['hot']} contributions"


@pytest.mark.gpu
@pytest.mark.parametrize("opt,B,steps", [("adam", 1 << 20, 3), ("adam", 256, 3), ("sgd", 1 << 20, 1)])
def test_bench_shape_steps(gpu, opt, B, steps):
    t0 = time.perf_counter()
    pr = _bench()
    st = I2vGpu(_bench_q(1), pr.planes, opt, 0.001 if opt == "adam" else 0.01)
    recs = []
    for s in range(steps):
        r, res = checked_step(st, s * B, B, B, f"bench {opt} B={B} step {s}", adam_step0=s, ref_device="cuda", with_res=True)
        print(f"  bench {opt} B={B} step {s}: {_hot(res)}")
        recs.append(r)
    report(f"i2v bench {opt} B={B}", recs)
    print(f"[i2v bench {opt} B={B}] {time.perf_counter() - t0:.1f} s")


@pytest.mark.gpu
def test_bench_shape_launch_loss_only_and_repeat(gpu):
    """a 4-step SGD launch (B = 2^20, last batch ragged) against four single launches (the launch bound sums the single steps'
    SGD half-widths); one loss-only call after an Adam step, which must leave Q, m and v alone; one B = 2^20 Adam step run
    twice from the same snapshot: the losses are bitwise equal, the tables and moments are not (the fp32 atomics of the
    gradient sums land in a different order), so that is reported, not asserted"""
    t0 = time.perf_counter()
    pr = _bench()
    B = 1 << 20
    n = 3 * B + 123457
    Q0 = _bench_q(2)
    multi, single = (I2vGpu(Q0, pr.planes, "sgd", 0.01) for _ in range(2))
    recs = launch_vs_singles(multi, single, n, B, 4)
    del multi, single
    st = I2vGpu(Q0, pr.planes, "adam", 0.001)
    recs.append(checked_step(st, 0, B, B, "adam step 0", ref_device="cuda"))
    recs.append(checked_step(st, B, B, B, "loss only (apply = 0)", adam_step0=1, apply=False, ref_device="cuda"))
    del st
    runs = []
    for _ in range(2):
        st = I2vGpu(Q0, pr.planes, "adam", 0.001)
        loss = st.run(0, B, B, 1)
        runs.append((loss, st.Q.clone(), *(m.clone() for m in st.mom["Q"])))
        del st
    same = [bool(np.array_equal(runs[0][0], runs[1][0]))] + [bool(torch.equal(a, b)) for a, b in zip(runs[0][1:], runs[1][1:])]
    d = (runs[0][1].to(F64) - runs[1][1].to(F64)).abs()
    print(f"  repeated B = 2^20 Adam step bitwise equal: loss {same[0]}, Q {same[1]}, m {same[2]}, v {same[3]}; "
          f"{int((d > 0).sum())} elements of Q differ, by at most {float(d.max()):.3g}")
    report("i2v bench launches", recs)
    print(f"[i2v bench launches] {time.perf_counter() - t0:.1f} s")


# ---------------------------------------------------------------- GPU: user embedding
def _crafted_csr(U, I, seed, long_row):
    """U users with 0 - 39 items (a quarter of them none) in random order, duplicates allowed, user 3 with long_row items"""
    rng = np.random.default_rng(seed)
    n = rng.integers(0, 40, U)
    n[rng.random(U) < 0.25] = 0
    n[3] = long_row
    row_ptr = np.concatenate([[0], np.cumsum(n)]).astype(np.int64)
    col = rng.integers(0, I, int(row_ptr[-1])).astype(np.int32)
    return torch.from_numpy(row_ptr).cuda(), torch.from_numpy(col).cuda()


@pytest.mark.gpu
def test_user_embedding_order(gpu):
    """the kernel adds in CSR order: rows (2^24, 1, -2^24) and its reverse sum to 0 and 1"""
    Q = torch.tensor([[2.0 ** 24], [1.0], [-(2.0 ** 24)]], device="cuda")
    row_ptr = torch.tensor([0, 3, 6, 6], device="cuda")
    col = torch.tensor([0, 1, 2, 2, 1, 0], dtype=torch.int32, device="cuda")
    P = torch.full((3, 1), 7.0, device="cuda")
    gpu.i2v_user_embedding(Q, row_ptr, col, P)
    assert P[:, 0].tolist() == [0.0, 1.0, 7.0]


@pytest.mark.gpu
@pytest.mark.parametrize("F", [1, 31, 32, 33, 100, 1024])
def test_user_embedding_sweep(gpu, F):
    U = resident_warps() + 1000
    I = 3001
    g = torch.Generator(device="cuda")
    g.manual_seed(F)
    Q = torch.randn(I, F, generator=g, device="cuda")
    P0 = torch.randn(U, F, generator=g, device="cuda")
    row_ptr, col = _crafted_csr(U, I, F, 9500)
    assert U > resident_warps()
    assert check_user_embedding(Q, row_ptr, col, P0, f"F={F}")["ok"]


@pytest.mark.gpu
def test_user_embedding_bench_shape(gpu):
    t0 = time.perf_counter()
    pr = _bench()
    row_ptr, col = pr.row_ptr, pr.col
    longest = int((row_ptr[1:] - row_ptr[:-1]).max())
    if longest <= 9000:                       # append a crafted user with 12 000 items in random order
        extra = torch.randperm(pr.I, device="cuda")[:12000].to(torch.int32)
        row_ptr = torch.cat([row_ptr, row_ptr[-1:] + extra.numel()])
        col = torch.cat([col, extra])
    U = row_ptr.numel() - 1
    assert U > resident_warps()
    Q = _bench_q(3)
    g = torch.Generator(device="cuda")
    g.manual_seed(4)
    P0 = torch.randn(U, BENCH_F, generator=g, device="cuda")
    print(f"  ML-20M CSR longest user row {longest}")
    assert check_user_embedding(Q, row_ptr, col, P0, "ML-20M F=100")["ok"]
    print(f"[i2v user embedding bench] {time.perf_counter() - t0:.1f} s")


# ---------------------------------------------------------------- GPU: through the class
class FitStepper(Stepper):
    """one Item2Vec.fit epoch as the launch side of launch_vs_singles"""
    device = "cuda"

    def __init__(self, model, loader, seed):
        self.model, self.loader, self.seed = model, loader, seed
        self.t = dict(Q=model.shared_embedding.weight)

    def run(self, lo, n, batch, k, adam_step0=0, apply=True, first_step=0):
        losses, orig = [], self.model._train_steps

        def rec(*a):
            out = orig(*a)
            losses.append(out.cpu().numpy())
            return out

        self.model._train_steps = rec
        torch.manual_seed(self.seed)
        self.model.fit(self.loader)
        self.model._train_steps = orig
        out = np.concatenate(losses)
        assert out.shape == (k,)
        return out

    def clean(self):
        ws = self.model._ws
        lay, _ = i2v_ws_layout(ws.I, ws.F, "adam")
        acc = views(ws.buf, lay, dict(gQ=torch.float32, cntI=torch.int64))
        torch.cuda.synchronize()
        return all(int(torch.count_nonzero(v)) == 0 for v in acc.values())


@pytest.mark.gpu
@pytest.mark.parametrize("opt,lr", [("adam", 0.001), ("sgd", 0.01)])
def test_fit_epoch_against_single_steps(gpu, opt, lr):
    """one fit epoch (one 256-step launch, the last batch ragged) against 256 single checked steps over the loader's order:
    each launch step's loss within the bound of the single step's reference, and under SGD the final table within the sum of
    the single steps' bounds.  Under Adam the final tables are not compared: its normalised updates amplify the last-bit
    differences that the fp32 atomics leave between two runs of the same steps, and over 256 steps they grow far beyond the sum
    of per-step bounds (two runs of the same single steps at this shape end up to 8.2e-6 apart, against 1.9e-9 under SGD)"""
    import logging
    from daisyrec_b200.model.AbstractRecommender import epoch_permutation
    from daisyrec_b200.model.Item2VecRecommender import Item2Vec
    from daisyrec_b200.utils.dataset import BasicDataset, get_dataloader
    t0 = time.perf_counter()
    pr = _bench()
    T, B = (1 << 16) - 100, 256
    rows = np.ascontiguousarray(pr.rows[:T].cpu().numpy().astype(np.int64))
    cfg = dict(gpu="0", user_num=pr.U, item_num=pr.I, factors=BENCH_F, train_ur={}, lr=lr, epochs=1,
               optimizer="default" if opt == "adam" else opt, init_method="default", early_stop=False, topk=50,
               logger=logging.getLogger("t"), progress=False, train_csr=(pr.row_ptr.cpu().numpy(), pr.col.cpu().numpy()))
    torch.manual_seed(0)
    model = Item2Vec(cfg)
    Q0 = model.shared_embedding.weight.clone()
    seed = 11
    torch.manual_seed(seed)
    perm = epoch_permutation(T, True).numpy()
    loader = get_dataloader(BasicDataset(rows), batch_size=B, shuffle=True, num_workers=0)
    multi = FitStepper(model, loader, seed)
    single = I2vGpu(Q0, rows[perm].T, opt, lr)
    k = -(-T // B)
    recs = launch_vs_singles(multi, single, T, B, k, states=opt == "sgd")
    d = (model.shared_embedding.weight.to(F64) - single.Q.to(F64)).abs()
    print(f"  fit epoch {opt}: {k} steps, last batch {T - (k - 1) * B} rows; worst single-step ratio "
          f"{max(r['ratio'] for r in recs[:-1]):.3g}, largest kappa needed {max(r['kneed'] for r in recs[:-1]):.3g}; "
          f"fit against singles: {int((d > 0).sum())} elements differ, by at most {float(d.max()):.3g}")
    report(f"i2v fit epoch {opt}", recs[-1:] + [r for r in recs[:-1] if not r["ok"]])
    assert all(r["ok"] for r in recs)
    print(f"[i2v fit epoch {opt}] {time.perf_counter() - t0:.1f} s")
