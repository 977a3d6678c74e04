"""The MF step's two opt-in modes, bit for bit: deterministic accumulation (ops.MFWorkspace(deterministic=True)) against an
exact host restatement of its fixed-point arithmetic, and the fused negative draws (ops.mf_bpr_train_steps_fused_neg)
against a host Philox4x32-10 and k-th-complement search.

Deterministic step, restated in numpy (det_step_host), exact for reg_2 = 0:
- scores: the device's own fp32 dot products (ops.mf_predict on the pre-step tables; predict and the step share row_geom and
  dot_rows);
- coefficient in fp32: BPR ex = float32(exp(-(float64) x)), sg = 1 / (1 + ex), c = -(sg (1 - sg)) / (1e-10 + sg); HL c = -1
  iff 1 - (pos - neg) >= 0; SL c = 2 (pos - y).  numpy's and CUDA's fp64 exp may differ by one fp64 ulp, which the rounding
  to fp32 hides unless the fp64 value lies within one ulp of an fp32 midpoint: such elements are counted and reported
  (expected: none);
- each contribution rounded to 2^-40 fixed point (np.rint, as __double2ll_rn) and summed exactly in int64;
- update: gd = fx / 2^40 + ca (sg + 0) + cb (sg + 0) in fp64, g = float32(gd), theta - float32(lr g).
The GPU cases compare with np.array_equal, no tolerance, teacher-forced (tables copied to the host before each checked
launch), and check that the fixed-point accumulators are zero after every launch.  With reg_1 = 0 the step loss is checked too
(det_loss_host: each triple's fp32 loss in 2^-24 fixed point): exactly under HL and SL, under BPR within -logf's last bit
per triple.  Adam, Adagrad and RMSprop take the exact
g and are checked on their own arithmetic: the fp64 update from that g and the device's pre-step moments, within a few fp32
ulps.  reg_2 != 0 (the batch norms in the regulariser) is checked against the fp64 oracle with the bound of
test_gpu_mf_step_fp64.py.

The triple-to-thread map (the index-tile size, DRB_TILE_CAP, read once per process) must not change anything: the same
launches in child processes at three tile caps give bitwise equal tables and losses, with reg_2 != 0, under every loss.
Before the step summed its loss and batch-norm partials per triple in fixed point (det_acc in step_kernel.cuh), the fp32
per-thread partials made the batch norms, and with reg_2 != 0 the tables, depend on that map.

Range: a table element's sum must stay below 2^23 = 8.4e6, the loss below 2^39 = 5.5e11 (2^-24 units), a batch-norm sum
below 2^31 = 2.1e9 (2^-32 units).  SL's and HL's losses are
unbounded, so the step checks every value and every integer addition and reports a run past either range as a non-finite loss
(the ValueError of the default mode), before the step is applied: test_det_out_of_range_is_reported.

Fused negatives: for the triple at plane position gt of step s, Philox4x32-10 with counter (gt lo, gt hi, s lo, s hi) and key
(seed lo, seed hi); k = (c0 n_comp) >> 32; item = k + #{s : col[s] - s <= k} over the user's sorted row.

The CPU tests pin the host Philox to Random123's known-answer vectors and show that each check rejects a defective stand-in.

Well-trained pairs: the fp32 coefficient is exactly 0 once 1 + exp(-x) rounds to 1 (x > 16.6), so the pairs of x >= 25 contribute
nothing.  Contributions near 2^-40 come from the last steps of the coefficient (x of 12 .. 17) times small elements, which
_trained_tables builds.

Measured on an H100 80GB HBM3 (132 SMs, 700 W power limit):
- bit-exact cases: every element equal in every case (F = 1 ... 1024 x BPR / HL / SL x reg_1 0 and 0.01, two launches each;
  the ML-20M shape at B = 2^20; the well-trained pairs).  No fp64 exp value lay within one ulp of an fp32 midpoint.  Every
  loss checked (reg_1 = 0) equal to det_loss_host, BPR's included (its slack went unused).
- fixed-point range (|table sum| < 2^23 = 8.4e6): the largest |sum| at the ML-20M shape was 1.24 under BPR (1.5e-7 of the
  range) and 5.5e3 under SL with labels 1 .. 5 and scores about 4 (6.5e-4 of the range).  A diverging SL run reaches further:
  the second step of the geometry cases at lr 0.05 reached 1.5e6 (0.18 of the range) at F = 100, and past the range at F = 128
  and above, where the step reported it; those cases now run SL at lr 0.002 (largest sum 5.3e4).
- optimisers under det, error / bound (OPT_ULPS = 8): Adam 0.47, Adagrad 0.49, RMSprop 0.48.
- reg_2 != 0 against the fp64 oracle at the ML-20M shape: error / bound 0.37 and 0.41 (kappa needed 1.3 and 3.5 of 134).  The
  losses equal the oracle's.  One fused launch on its own negatives: 0.77 (kappa 4.2).
- tile caps 512 (default), 256 and 1024 at the ML-20M shape: all seven cases give bitwise equal tables and losses.  With the
  parent commit's fp32 scalar partials, three of the six reg_2 != 0 cases differed: BPR / SGD at cap 256 (the user table and
  one item element), BPR / Adam and TL at cap 1024 (one item element each).  The reg_2 = 0 case was equal.
Stand-ins (CPU cases, fresh / well-trained tables), share of table elements changed: truncation 0 / 7.1 %, a 2^-39 scale
(quantised and read back at 2^-39) 0 / 7.1 %, accumulators kept across steps 100 % / 76 %, fp32 expf 4.7 % / 0, lr g fused
into the subtraction 4.3 % / 0.
Share of fused draws changed: % n_comp 95 %, step word 0 95 % (steps 2 .. 4), complement search off by one 5.2 %.
"""
import hashlib
import os
import subprocess
import sys
import time

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)

F32 = np.float32
TWO40 = 2.0 ** 40
ML20M = (138_493, 26_744, 64, 1 << 20)          # the bench's MF shape and batch
GEOM_F = [1, 2, 6, 8, 32, 64, 100, 128, 512, 1024]   # every row_geom: VEC 1 / 2 / 4, W x NCH up to 32 x 8
U_RND = 2.0 ** -24


# ---------------------------------------------------------------- the deterministic step, restated
def coef(loss, pos, neg, exp64=True):
    """fp32 coefficients d loss / d pos, d loss / d neg of the step (pair_loss in step_kernel.cuh) and the count of fp64 exp
    values within one fp64 ulp of an fp32 rounding midpoint (BPR)"""
    pos, neg = np.asarray(pos, F32), np.asarray(neg, F32)
    near = 0
    if loss == "BPR":
        x = pos - neg
        if exp64:
            e = np.exp(-x.astype(np.float64))
            ex = e.astype(F32)
            up, dn = np.nextafter(ex, F32(np.inf)), np.nextafter(ex, F32(0))
            for nb in (up, dn):
                mid = (ex.astype(np.float64) + nb.astype(np.float64)) / 2
                near += int((np.abs(e - mid) <= np.spacing(e)).sum())
        else:
            ex = np.exp(-x)                                # fp32 exp: the stand-in of the non-det coefficient
        sg = F32(1) / (F32(1) + ex)
        c = -(sg * (F32(1) - sg)) / (F32(1e-10) + sg)
        return c, -c, near
    if loss == "HL":
        m = F32(1) - (pos - neg)
        c = np.where(m >= 0, F32(-1), F32(0)).astype(F32)
        return c, -c, 0
    if loss == "SL":
        c = F32(2) * (pos - neg)
        return c, np.zeros_like(c), 0
    raise ValueError(loss)


def _rowsum(idx, vals, out):
    """out[idx[t]] += vals[t] exactly (int64 rows)"""
    order = np.argsort(idx, kind="stable")
    s = idx[order]
    starts = np.flatnonzero(np.r_[True, s[1:] != s[:-1]])
    out[s[starts]] += np.add.reduceat(vals[order], starts, axis=0)


def det_fixed(P, Q, bu, bi, bj, loss, pos, neg, scale=TWO40, rnd=np.rint, exp64=True, chunk=1 << 17):
    """-> dict(fxP [U, F], fxQ [I, F] int64 fixed-point gradient sums; cu [U], ci [I], cj [I] occurrence counts; near):
    phase 1 of the deterministic step (pw losses: bj holds labels, no j row, no j count)"""
    pw = loss in ("CL", "SL")
    fxP, fxQ = np.zeros(P.shape, np.int64), np.zeros(Q.shape, np.int64)
    q = lambda v: rnd(v.astype(np.float64) * scale).astype(np.int64)
    near = 0
    for a in range(0, len(bu), chunk):
        b = min(len(bu), a + chunk)
        u, i, j = bu[a:b], bi[a:b], bj[a:b]
        c, cn, nr = coef(loss, pos[a:b], neg[a:b], exp64)
        near += nr
        c, cn = c[:, None], cn[:, None]
        p, qi = P[u], Q[i]
        if loss == "BPR":
            qj = Q[j]
            gu, gi = c * (qi - qj), c * p
            gj = -gi
        else:
            qj = np.zeros_like(qi) if pw else Q[j]
            gu, gi, gj = c * qi + cn * qj, c * p, cn * p
        _rowsum(u, q(gu), fxP)
        _rowsum(i, q(gi), fxQ)
        if not pw:
            _rowsum(j, q(gj), fxQ)
    cu = np.bincount(bu, minlength=len(P))
    ci = np.bincount(bi, minlength=len(Q))
    cj = np.zeros(len(Q), np.int64) if pw else np.bincount(bj, minlength=len(Q))
    return dict(fxP=fxP, fxQ=fxQ, cu=cu, ci=ci, cj=cj, near=near)


def det_grad(T, fx, ca, cb, reg1, scale=TWO40):
    """fp32 gradient of every row (0 where untouched) and the touched mask: the DET sweep's fp64 assembly, rounded once"""
    touched = (ca + cb) > 0
    sg = (F32(reg1) * np.sign(T).astype(F32)).astype(np.float64)
    gd = fx / scale + (ca[:, None].astype(np.float64) * (sg + 0.0) + cb[:, None].astype(np.float64) * (sg + 0.0))
    gd[~touched] = 0.0
    return gd.astype(F32), touched


def det_sgd(T, g, touched, lr, fused=False):
    out = T.copy()
    if fused:       # stand-in: lr g folded into the subtraction (one rounding)
        out[touched] = (T[touched].astype(np.float64) - np.float64(F32(lr)) * g[touched].astype(np.float64)).astype(F32)
    else:
        out[touched] = T[touched] - F32(lr) * g[touched]
    return out


def det_step_host(P, Q, bu, bi, bj, loss, pos, neg, lr, reg1, scale=TWO40, rnd=np.rint, exp64=True, fused=False,
                  carry=None):
    """one deterministic SGD step (reg_2 = 0) -> (P', Q', fixed-point sums used).  carry: a previous step's sums added to
    this step's (the stand-in of accumulators not cleared between steps)."""
    d = det_fixed(P, Q, bu, bi, bj, loss, pos, neg, scale, rnd, exp64)
    if carry is not None:
        d["fxP"] = d["fxP"] + carry["fxP"]
        d["fxQ"] = d["fxQ"] + carry["fxQ"]
    gP, tP = det_grad(P, d["fxP"], d["cu"], np.zeros_like(d["cu"]), reg1, scale)
    gQ, tQ = det_grad(Q, d["fxQ"], d["ci"], d["cj"], reg1, scale)
    return det_sgd(P, gP, tP, lr, fused), det_sgd(Q, gQ, tQ, lr, fused), d


def host_scores(P, Q, u, i):
    """fp32 scores for the CPU cases (the GPU cases take the device's own)"""
    return np.einsum("nf,nf->n", P[u].astype(np.float64), Q[i].astype(np.float64)).astype(F32)


# ---------------------------------------------------------------- Philox4x32-10 and the fused negative draw, restated
_M = 0xFFFFFFFF


def philox4x32(c0, c1, c2, c3, k0, k1):
    """vectorised Philox4x32-10 (philox_round / philox4x32 in common.cuh): uint32 arrays, scalar key words"""
    c = [np.asarray(x, np.uint64) & _M for x in (c0, c1, c2, c3)]
    k0, k1 = int(k0) & _M, int(k1) & _M
    for _ in range(10):
        p0 = c[0] * np.uint64(0xD2511F53)
        p1 = c[2] * np.uint64(0xCD9E8D57)
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & np.uint64(_M), p1 >> np.uint64(32), p1 & np.uint64(_M)
        c = [hi1 ^ c[1] ^ np.uint64(k0), lo1, hi0 ^ c[3] ^ np.uint64(k1), lo0]
        k0 = (k0 + 0x9E3779B9) & _M
        k1 = (k1 + 0xBB67AE85) & _M
    return [x.astype(np.uint32) for x in c]


def draw_negatives(row_ptr, col, I, seed, users, gt, step, kmap="mulhi", step_word=True, search="le", k=None):
    """host draw_negative for triples (users, plane positions gt, steps).  Stand-ins: kmap='mod' (k = c0 % n_comp),
    step_word=False (counter words 2, 3 left at 0), search='lt' (col[s] - s < k: the complement search off by one).
    k (optional): the complement ranks themselves, in place of the Philox draw (seed, gt and step are then unused)."""
    users = np.asarray(users, np.int64)
    deg = np.diff(row_ptr)
    if k is None:
        gt = np.asarray(gt, np.uint64)
        step = np.broadcast_to(np.asarray(step, np.uint64), gt.shape)
        if not step_word:
            step = np.zeros_like(step)
        w = philox4x32(gt & np.uint64(_M), gt >> np.uint64(32), step & np.uint64(_M), step >> np.uint64(32), seed & _M,
                       seed >> 32)
        n_comp = (I - deg[users]).astype(np.uint64)
        c0 = w[0].astype(np.uint64)
        k = (c0 % n_comp) if kmap == "mod" else ((c0 * n_comp) >> np.uint64(32))
    k = np.asarray(k).astype(np.int64)
    # d[s] = col[s] - (s - row start) is non-decreasing along a row: count #{d <= k} by one search over (row, d) keys
    row_of = np.repeat(np.arange(len(row_ptr) - 1, dtype=np.int64), deg)
    d = col.astype(np.int64) - (np.arange(len(col), dtype=np.int64) - row_ptr[row_of])
    keys = row_of * (1 << 32) + d
    cnt = np.searchsorted(keys, users * (1 << 32) + k, side="right" if search == "le" else "left") - row_ptr[users]
    item = k + cnt
    return np.minimum(item, I - 1).astype(np.int32)


def csr(rows, I):
    """sorted CSR (row_ptr int64, col int32) from a list of item lists"""
    rows = [np.unique(np.asarray(r, np.int64)) for r in rows]
    row_ptr = np.zeros(len(rows) + 1, np.int64)
    row_ptr[1:] = np.cumsum([len(r) for r in rows])
    col = np.concatenate(rows).astype(np.int32) if rows else np.zeros(0, np.int32)
    return row_ptr, col


def crafted_csr(seed=5):
    """users: 0 no row (n_comp = I); 1 missing one middle item; 2 missing only item 0; 3 missing only item I - 1; 4 a hub
    row longer than 2^16; 5 .. 63 random rows"""
    rng = np.random.default_rng(seed)
    I = 70_000
    every = np.arange(I)
    rows = [[], np.delete(every, 31_337), every[1:], every[:-1], rng.choice(I, 66_000, replace=False)]
    rows += [rng.choice(I, int(rng.integers(1, 400)), replace=False) for _ in range(59)]
    return I, *csr(rows, I)


# ---------------------------------------------------------------- CPU checks: the restatements and their stand-ins
def test_philox_known_answers():
    """Random123's kat_vectors for philox4x32_10"""
    z = np.zeros(1, np.uint32)
    got = [int(x[0]) for x in philox4x32(z, z, z, z, 0, 0)]
    assert got == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    f = np.full(1, 0xFFFFFFFF, np.uint32)
    got = [int(x[0]) for x in philox4x32(f, f, f, f, 0xFFFFFFFF, 0xFFFFFFFF)]
    assert got == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]
    c = [np.array([v], np.uint32) for v in (0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344)]
    got = [int(x[0]) for x in philox4x32(*c, 0xA4093822, 0x299F31D0)]
    assert got == [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1]


def test_kth_complement_is_the_sorted_complement():
    """draw_negatives' search over every rank k in [0, n_comp) of each user is the user's complement in ascending order;
    the off-by-one stand-in is not"""
    I, row_ptr, col = crafted_csr()
    bad = 0
    for u in range(len(row_ptr) - 1):
        want = np.setdiff1d(np.arange(I), col[row_ptr[u]:row_ptr[u + 1]])
        k = np.arange(len(want))
        users = np.full(len(k), u)
        assert np.array_equal(draw_negatives(row_ptr, col, I, 0, users, None, None, k=k), want), u
        bad += not np.array_equal(draw_negatives(row_ptr, col, I, 0, users, None, None, search="lt", k=k), want)
    # the stand-in agrees only on an empty row and on rows that are a tail of the item range, where no k reaches col[s] - s
    assert bad >= len(row_ptr) - 4, bad


def _fused_case_cpu(seed=3, B=4096, steps=3, first=2):
    I, row_ptr, col = crafted_csr()
    rng = np.random.default_rng(seed)
    n = (first + steps) * B
    users = rng.integers(len(row_ptr) - 1, size=n)
    gt = np.arange(first * B, n, dtype=np.uint64)
    return I, row_ptr, col, users, gt, gt // np.uint64(B)


def test_draw_negatives_host_properties_and_standins():
    I, row_ptr, col, users, gt, step = _fused_case_cpu()
    seed = (1 << 40) + 12345
    u = users[gt.astype(np.int64)]
    j = draw_negatives(row_ptr, col, I, seed, u, gt, step)
    pos = set(zip(np.repeat(np.arange(len(row_ptr) - 1), np.diff(row_ptr)).tolist(), col.tolist()))
    assert not any((int(a), int(b)) in pos for a, b in zip(u, j))
    assert (j[u == 1] == 31_337).all() and (j[u == 2] == 0).all() and (j[u == 3] == I - 1).all()
    # the empty row covers the item range uniformly: its last item is reachable
    e = j[u == 0]
    assert e.min() < I // 50 and e.max() > I - I // 50
    fracs = {}
    for name, kw in (("mod", dict(kmap="mod")), ("step0", dict(step_word=False)), ("off-by-one", dict(search="lt"))):
        fracs[name] = float((draw_negatives(row_ptr, col, I, seed, u, gt, step, **kw) != j).mean())
        assert fracs[name] > 0, name
    print("fused-draw stand-ins, share of draws changed:", fracs)


def _trained_tables(rng, U, I, F, planes):
    """tables on which the triples of `planes` score x = p.(q_i - q_j) of about 12 .. 17, well-trained pairs: the fp32
    coefficient runs down its last steps (1 - sg is a multiple of 2^-24) to exactly 0 beyond x = 16.6.  The items' last F / 8
    elements are of order 1e-5 and the users' are 0, so on those elements the user contributions c (q_i - q_j) lie between
    0 and a few dozen units of 2^-40, and the update of a zero element, -lr float32(fx 2^-40), shows the sum to the unit."""
    bu, bi, bj = planes
    t = F - F // 8
    P = (np.full((U, F), 0.5, F32) * rng.uniform(0.85, 1.2, size=(U, 1))).astype(F32)
    P[:, t:] = 0
    Q = np.full((I, F), -0.2, F32) + (rng.standard_normal((I, F)) * 0.02).astype(F32)
    ui = np.unique(bi)
    Q[ui] = (np.full((F,), 0.3, F32) + rng.standard_normal((len(ui), F)) * 0.02).astype(F32)
    Q[:, t:] = (rng.standard_normal((I, F - t)) * 1e-5).astype(F32)
    return P, Q


def _cpu_case(rng, U, I, F, B, trained=False):
    bu = rng.integers(U, size=B).astype(np.int32)
    bi = (rng.random(B) ** 2 * (I // 2)).astype(np.int32)                      # positives among the first half
    bj = (I // 2 + rng.integers(I - I // 2, size=B)).astype(np.int32)          # negatives among the second
    if trained:
        P, Q = _trained_tables(rng, U, I, F, (bu, bi, bj))
    else:
        P, Q = (rng.standard_normal((U, F)) * 0.1).astype(F32), (rng.standard_normal((I, F)) * 0.1).astype(F32)
    return P, Q, bu, bi, bj


def test_det_restatement_rejects_standins():
    """truncation, a 2^-39 scale, accumulators kept across steps, fp32 expf, lr g fused into the subtraction: each changes
    the restated tables of at least one case (the shares are printed)"""
    rng = np.random.default_rng(7)
    cases = {"fresh": _cpu_case(rng, 2000, 1000, 64, 1 << 15), "trained": _cpu_case(rng, 2000, 1000, 64, 1 << 15, True)}
    lr, reg1 = 0.01, 0.0
    share = {}
    for name, (P, Q, bu, bi, bj) in cases.items():
        pos, neg = host_scores(P, Q, bu, bi), host_scores(P, Q, bu, bj)
        if name == "trained":
            x = pos - neg
            assert 12 < np.median(x) < 17
        P1, Q1, d1 = det_step_host(P, Q, bu, bi, bj, "BPR", pos, neg, lr, reg1)
        # step 2 from the new tables: the stale stand-in adds step 1's sums
        pos2, neg2 = host_scores(P1, Q1, bu, bi), host_scores(P1, Q1, bu, bj)
        P2, Q2, _ = det_step_host(P1, Q1, bu, bi, bj, "BPR", pos2, neg2, lr, reg1)
        standins = {
            "trunc": lambda: det_step_host(P, Q, bu, bi, bj, "BPR", pos, neg, lr, reg1, rnd=np.trunc)[:2],
            "scale 2^-39 both ways": lambda: det_step_host(P, Q, bu, bi, bj, "BPR", pos, neg, lr, reg1, scale=2.0 ** 39)[:2],
            "stale": lambda: det_step_host(P1, Q1, bu, bi, bj, "BPR", pos2, neg2, lr, reg1, carry=d1)[:2],
            "expf32": lambda: det_step_host(P, Q, bu, bi, bj, "BPR", pos, neg, lr, reg1, exp64=False)[:2],
            "fused lr g": lambda: det_step_host(P, Q, bu, bi, bj, "BPR", pos, neg, lr, reg1, fused=True)[:2],
        }
        for s, f in standins.items():
            gP, gQ = f()
            rP, rQ = (P2, Q2) if s == "stale" else (P1, Q1)
            share[(name, s)] = float(np.concatenate([(gP != rP).ravel(), (gQ != rQ).ravel()]).mean())
    print("det stand-ins, share of table elements changed:", {f"{a}/{b}": v for (a, b), v in share.items()})
    for s in ("trunc", "scale 2^-39 both ways", "stale", "expf32", "fused lr g"):
        assert max(share[("fresh", s)], share[("trained", s)]) > 0, s


def test_det_restatement_hand_computed():
    """one triple, F = 2: the fixed-point sums and the update worked by hand"""
    P = np.array([[0.5, -0.25]], F32)
    Q = np.array([[0.25, 0.5], [-0.5, 0.125]], F32)
    bu, bi, bj = np.array([0], np.int32), np.array([0], np.int32), np.array([1], np.int32)
    pos, neg = host_scores(P, Q, bu, bi), host_scores(P, Q, bu, bj)
    assert pos[0] == F32(0.0) and neg[0] == F32(-0.28125)
    x = F32(0.28125)
    sg = F32(1) / (F32(1) + F32(np.exp(-np.float64(x))))
    c = -(sg * (F32(1) - sg)) / (F32(1e-10) + sg)
    P1, Q1, d = det_step_host(P, Q, bu, bi, bj, "BPR", pos, neg, 0.5, 0.0)
    assert d["fxP"][0, 0] == np.rint(np.float64(c * F32(0.75)) * TWO40)
    assert d["fxQ"][1, 1] == np.rint(np.float64(-(c * F32(-0.25))) * TWO40)
    assert P1[0, 0] == P[0, 0] - F32(0.5) * F32(d["fxP"][0, 0] / TWO40)


# ---------------------------------------------------------------- GPU plumbing
def _torch_ops():
    import torch
    from daisyrec_b200 import ops
    return torch, ops


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _align(n):
    return (n + 255) // 256 * 256


def ws_views(ws):
    """int64 / float32 views of a deterministic MF workspace (mirrors carve in step.cuh): dict(gP64, gQ64, accfx, mP, vP, mQ,
    vQ) (None where the optimiser keeps no such table)"""
    import torch
    U, I, F, opt = ws.U, ws.I, ws.F, ws.opt
    off = _align(256)
    out = {}
    for name, n in (("gP", 4 * U * F), ("gQ", 4 * I * F), ("cntU", 4 * U), ("cntI", 8 * I)):
        out[name] = (off, n)
        off += _align(n)
    for name, on in (("mP", opt != 0), ("vP", opt == 1), ("mQ", opt != 0), ("vQ", opt == 1)):
        if on:
            out[name] = (off, 4 * (U if name.endswith("P") else I) * F)
            off += _align(out[name][1])
    for name, n in (("gP64", 8 * U * F), ("gQ64", 8 * I * F), ("accfx", 64)):
        out[name] = (off, n)
        off += _align(n)
    assert off == ws.buf.numel(), (off, ws.buf.numel())
    views = {}
    for name, (o, n) in out.items():
        dt = torch.int64 if name in ("gP64", "gQ64", "accfx", "cntI") else torch.float32
        views[name] = ws.buf[o:o + n].view(dt)
    for name in ("mP", "vP", "mQ", "vQ"):
        views.setdefault(name, None)
    return views


def ws_fixed_zero(ws):
    v = ws_views(ws)
    return all(int(v[k].count_nonzero()) == 0 for k in ("gP64", "gQ64", "accfx", "gP", "gQ", "cntU", "cntI"))


class DetRun:
    """device tables + a deterministic workspace; one teacher-forced launch at a time"""

    def __init__(self, P, Q, opt="sgd"):
        torch, ops = _torch_ops()
        self.torch, self.ops, self.opt = torch, ops, opt
        self.P, self.Q = _dev(P), _dev(Q)
        self.ws = ops.MFWorkspace(P.shape[0], Q.shape[0], P.shape[1], opt, "cuda", deterministic=True)

    def tables(self):
        self.torch.cuda.synchronize()
        return self.P.cpu().numpy(), self.Q.cpu().numpy()

    def scores(self, bu, bi):
        return self.ops.mf_predict(self.P, self.Q, _dev(bu), _dev(bi)).cpu().numpy()

    def launch(self, planes, batch, k, lr, reg1, reg2, loss="BPR", first=0, adam_step0=0):
        hp = self.ops.hyper(lr, reg1, reg2, self.opt, loss=loss)
        bu, bi, bj = (_dev(x) for x in planes)
        out = self.ops.mf_bpr_train_steps(self.P, self.Q, self.ws, bu, bi, bj, batch, first, k, hp, adam_step0=adam_step0)
        return out.cpu().numpy()


ACC_SCALE = 2.0 ** 24      # kDetAccScale: the step's scalar sums


def det_loss_host(loss, pos, neg):
    """the step loss for reg_1 = reg_2 = 0: each triple's fp32 loss (pair_loss) in 2^-24 fixed point, summed exactly, the
    total rounded to fp32 -> (loss, slack).  HL and SL are exact (slack 0).  BPR's -logf may differ from the correctly
    rounded log by an fp32 ulp per triple: the slack covers that and the final rounding."""
    pos, neg = np.asarray(pos, F32), np.asarray(neg, F32)
    if loss == "HL":
        m = F32(1) - (pos - neg)
        t = np.where(m > 0, m, F32(0)).astype(F32)
    elif loss == "SL":
        d = pos - neg
        t = d * d
    else:
        sg = F32(1) / (F32(1) + np.exp(-(pos - neg).astype(np.float64)).astype(F32))
        t = (-np.log((F32(1e-10) + sg).astype(np.float64))).astype(F32)
    fx = int(np.rint(t.astype(np.float64) * ACC_SCALE).astype(np.int64).sum())
    total = F32(fx / ACC_SCALE)
    slack = 0.0 if loss != "BPR" else float(np.spacing(t).astype(np.float64).sum() + len(t) / ACC_SCALE + np.spacing(total))
    return total, slack


def exact_case(run, planes, loss, lr, reg1):
    """one single-step launch against det_step_host on the pre-step tables -> (ok, record); with reg_1 = 0 the step loss
    is checked against det_loss_host as well"""
    bu, bi, bj = planes
    P, Q = run.tables()
    pos = run.scores(bu, bi)
    neg = bj.astype(F32) if loss in ("CL", "SL") else run.scores(bu, bj)
    rP, rQ, d = det_step_host(P, Q, bu, bi, bj, loss, pos, neg, lr, reg1)
    got_loss = float(run.launch(planes, len(bu), 1, lr, reg1, 0.0, loss)[0])
    gP, gQ = run.tables()
    zero = ws_fixed_zero(run.ws)
    fxmax = max(int(np.abs(d["fxP"]).max()), int(np.abs(d["fxQ"]).max())) / TWO40
    rec = dict(loss=loss, reg1=reg1, diffP=int((gP != rP).sum()), diffQ=int((gQ != rQ).sum()), near=d["near"], zero=zero,
               fxmax=fxmax, moved=float(np.concatenate([(gP != P).ravel(), (gQ != Q).ravel()]).mean()))
    ok = np.array_equal(gP, rP) and np.array_equal(gQ, rQ) and zero
    if reg1 == 0:
        want, slack = det_loss_host(loss, pos, neg)
        rec["loss_err"], rec["loss_slack"] = abs(got_loss - float(want)), slack
        ok = ok and rec["loss_err"] <= slack
    return ok, rec


def zipf_planes(rng, U, I, n, loss="BPR", labels=5):
    bu = np.minimum(U - 1, rng.zipf(1.3, size=n) - 1).astype(np.int32)
    bi = (rng.random(n) ** 2 * I).astype(np.int32)
    bj = rng.integers(labels + 1, size=n).astype(np.int32) if loss in ("CL", "SL") else rng.integers(I, size=n).astype(np.int32)
    if loss == "CL":
        bj = np.minimum(bj, 1).astype(np.int32)
    return bu, bi, bj


# ---------------------------------------------------------------- GPU: deterministic mode, bit for bit
@pytest.mark.gpu
@pytest.mark.parametrize("F", GEOM_F)
def test_det_sgd_bit_exact_every_geometry(F):
    """BPR, HL and SL under SGD with reg_2 = 0, reg_1 0 and 0.01: two teacher-forced launches each, np.array_equal"""
    U, I, B = 300, 200, 4096
    bad = []
    for loss in ("BPR", "HL", "SL"):
        for reg1 in (0.0, 0.01):
            rng = np.random.default_rng(F * 10 + len(loss))
            P0, Q0 = (rng.standard_normal((U, F)) * 0.3).astype(F32), (rng.standard_normal((I, F)) * 0.3).astype(F32)
            run = DetRun(P0, Q0)
            for s in range(2):
                # SL at lr 0.05 diverges in its second step at F >= 128 (and is then reported as out of range)
                ok, rec = exact_case(run, zipf_planes(rng, U, I, B, loss), loss, 0.002 if loss == "SL" else 0.05, reg1)
                print(F, s, rec)
                assert rec["moved"] > 0.3, rec
                if not ok:
                    bad.append((s, rec))
    assert not bad, bad


def ml20m_positives(seed=2022):
    """(coo_u, coo_i, row_ptr, col) of the bench's synthetic ML-20M interactions, on the host"""
    from daisyrec_b200.utils.synthetic import make_interactions
    U, I = ML20M[:2]
    d = make_interactions(U, I, 20_000_000, seed=seed, device="cuda")
    return tuple(d[k].cpu().numpy() for k in ("coo_u", "coo_i", "row_ptr", "col"))


_ML = {}


def ml20m_batches(n_batches, loss="BPR", seed=11):
    """n_batches bench batches of (user, positive, uniform negative) -- or (user, item, label) -- triples drawn from the
    synthetic ML-20M interactions"""
    if "pos" not in _ML:
        _ML["pos"] = ml20m_positives()
    cu, ci = _ML["pos"][:2]
    U, I, F, B = ML20M
    rng = np.random.default_rng(seed)
    sel = rng.integers(len(cu), size=n_batches * B)
    bj = rng.integers(I, size=n_batches * B).astype(np.int32)
    if loss in ("CL", "SL"):
        bj = rng.integers(1, 6, size=n_batches * B).astype(np.int32) if loss == "SL" else rng.integers(2, size=n_batches * B).astype(np.int32)
    return cu[sel].astype(np.int32), ci[sel].astype(np.int32), bj


@pytest.mark.gpu
def test_det_sgd_bit_exact_ml20m_shape():
    """the bench shape and batch: BPR with reg_1 0.001 over two launches, and SL with ratings 1 .. 5 as labels on tables
    whose scores are of the labels' size (the largest fixed-point sums); records the range margin"""
    U, I, F, B = ML20M
    rng = np.random.default_rng(1)
    out = []
    for loss, scale in (("BPR", 0.01), ("SL", 0.25)):
        P0, Q0 = (rng.standard_normal((U, F)) * scale).astype(F32), (rng.standard_normal((I, F)) * scale).astype(F32)
        if loss == "SL":
            P0 += F32(0.25)
            Q0 += F32(0.25)                                  # scores about F / 16 = 4
        run = DetRun(P0, Q0)
        bu, bi, bj = ml20m_batches(2, loss)
        for s in range(2 if loss == "BPR" else 1):          # SL at lr 0.01 on these tables diverges in its second step
            pl = tuple(x[s * B:(s + 1) * B] for x in (bu, bi, bj))
            ok, rec = exact_case(run, pl, loss, 0.01, 0.001)
            rec["range_margin"] = 2.0 ** 23 / rec["fxmax"]
            print("ml20m", s, rec)
            out.append((ok, rec))
    assert all(ok for ok, _ in out), [r for _, r in out]


@pytest.mark.gpu
def test_det_sgd_bit_exact_well_trained_pairs():
    """well-trained pairs (x about 12 .. 17, see _trained_tables): contributions of a few units of 2^-40 and below"""
    rng = np.random.default_rng(3)
    U, I, F, B = 2000, 1000, 64, 1 << 16
    P, Q, bu, bi, bj = _cpu_case(rng, U, I, F, B, trained=True)
    run = DetRun(P, Q)
    pos, neg = run.scores(bu, bi), run.scores(bu, bj)
    assert 12 < np.median(pos - neg) < 17
    ok, rec = exact_case(run, (bu, bi, bj), "BPR", 0.05, 0.0)
    print("trained", rec)
    assert rec["moved"] > 0 and ok, rec


@pytest.mark.gpu
@pytest.mark.parametrize("opt", ["sgd", "adam"])
def test_det_multistep_launch_equals_single_launches(opt):
    """a 4-step launch at first_step 1 == four single-step launches, bitwise (tables, losses, moments), reg_2 != 0"""
    rng = np.random.default_rng(5)
    U, I, F, B = 5000, 700, 64, 8192
    P0, Q0 = (rng.standard_normal((U, F)) * 0.1).astype(F32), (rng.standard_normal((I, F)) * 0.1).astype(F32)
    planes = zipf_planes(rng, U, I, 5 * B)
    a, b = DetRun(P0, Q0, opt), DetRun(P0, Q0, opt)
    la = a.launch(planes, B, 4, 0.01, 0.001, 0.01, first=1, adam_step0=0)
    lb = np.concatenate([b.launch(planes, B, 1, 0.01, 0.001, 0.01, first=1 + s, adam_step0=s) for s in range(4)])
    (Pa, Qa), (Pb, Qb) = a.tables(), b.tables()
    assert np.array_equal(Pa, Pb) and np.array_equal(Qa, Qb)
    assert np.array_equal(la, lb), (la, lb)
    va, vb = ws_views(a.ws), ws_views(b.ws)
    for k in ("mP", "vP", "mQ", "vQ"):
        if va[k] is not None:
            assert a.torch.equal(va[k], vb[k]), k
    assert ws_fixed_zero(a.ws) and ws_fixed_zero(b.ws)
    assert not np.array_equal(Pa, P0)


@pytest.mark.gpu
def test_det_fit_steps_per_launch_is_bitwise_neutral():
    import logging
    import torch
    from daisyrec_b200.model.MFRecommender import MF
    from daisyrec_b200.utils.dataset import BasicDataset, get_dataloader
    rng = np.random.default_rng(9)
    U, I, T, B = 700, 400, 30_000, 1024
    data = np.stack([np.minimum(U - 1, rng.zipf(1.3, size=T) - 1), rng.integers(I, size=T), rng.integers(I, size=T)],
                    1).astype(np.int32)
    runs = []
    for spl in (1, 0):
        cfg = dict(gpu='0', seed=2022, topk=50, cand_num=1000, sample_method='uniform', sample_ratio=0, num_ng=4,
                   batch_size=B, loss_type='BPR', init_method='default', optimizer='adam', early_stop=False,
                   UID_NAME='user', IID_NAME='item', INTER_NAME='rating', TID_NAME='timestamp', user_num=U, item_num=I,
                   factors=64, epochs=2, lr=0.01, reg_1=0.001, reg_2=0.001, logger=logging.getLogger('t'), progress=False,
                   deterministic=True, steps_per_launch=spl)
        torch.manual_seed(7)
        m = MF(cfg)
        m.fit(get_dataloader(BasicDataset(data), batch_size=B, shuffle=False))
        runs.append((m.embed_user.weight.cpu().numpy(), m.embed_item.weight.cpu().numpy()))
    assert np.array_equal(runs[0][0], runs[1][0]) and np.array_equal(runs[0][1], runs[1][1])


def _opt_ref(opt, theta, g, m, v, lr, t, beta1=0.9, beta2=0.999, eps=1e-8):
    """fp64 update from the exact fp32 gradient and the device's fp32 pre-step moments (the kernel's fp32 constants) ->
    (theta', magnitude of the update's terms for the bound)"""
    th, g, m = theta.astype(np.float64), g.astype(np.float64), m.astype(np.float64)
    if opt == "adam":
        b1c, b2c = np.float64(F32(1) - F32(beta1)), np.float64(F32(1) - F32(beta2))
        v = v.astype(np.float64)
        step = np.float64(F32(np.float64(F32(lr)) / (1.0 - np.float64(F32(beta1)) ** t)))
        bc2 = np.float64(F32(np.sqrt(1.0 - np.float64(F32(beta2)) ** t)))
        m1 = m + (g - m) * b1c
        v1 = v * np.float64(F32(beta2)) + b2c * g * g
        den = np.sqrt(v1) / bc2 + np.float64(F32(eps))
        return th - step * (m1 / den), step * (np.abs(m) + np.abs(g)) / den
    if opt == "adagrad":
        ss = m + g * g
        den = np.sqrt(ss) + np.float64(F32(1e-10))
        return th - np.float64(F32(lr)) * (g / den), np.float64(F32(lr)) * np.abs(g) / den
    sq = m * np.float64(F32(0.99)) + np.float64(F32(1) - F32(0.99)) * g * g
    den = np.sqrt(sq) + np.float64(F32(1e-8))
    return th - np.float64(F32(lr)) * (g / den), np.float64(F32(lr)) * np.abs(g) / den


OPT_ULPS = 8.0      # |device - fp64| <= 2 u |theta| + OPT_ULPS u (update terms)


@pytest.mark.gpu
@pytest.mark.parametrize("opt", ["adam", "adagrad", "rmsprop"])
def test_det_optimisers_on_the_exact_gradient(opt):
    """reg_2 = 0: the gradient is det_step_host's, exactly; the optimiser's fp32 arithmetic is checked alone against fp64,
    three teacher-forced launches (moments nonzero from the second on)"""
    rng = np.random.default_rng(13)
    U, I, F, B, lr = 3000, 500, 64, 8192, 0.01
    P0, Q0 = (rng.standard_normal((U, F)) * 0.1).astype(F32), (rng.standard_normal((I, F)) * 0.1).astype(F32)
    run = DetRun(P0, Q0, opt)
    worst = 0.0
    for s in range(3):
        bu, bi, bj = zipf_planes(rng, U, I, B)
        P, Q = run.tables()
        vw = ws_views(run.ws)
        mom = {k: (vw[k].cpu().numpy().reshape(-1, F) if vw[k] is not None else None) for k in ("mP", "vP", "mQ", "vQ")}
        d = det_fixed(P, Q, bu, bi, bj, "BPR", run.scores(bu, bi), run.scores(bu, bj))
        gP, _ = det_grad(P, d["fxP"], d["cu"], np.zeros_like(d["cu"]), 0.001)
        gQ, _ = det_grad(Q, d["fxQ"], d["ci"], d["cj"], 0.001)
        run.launch((bu, bi, bj), B, 1, lr, 0.001, 0.0, adam_step0=s)
        nP, nQ = run.tables()
        for T, g, got, m, v in ((P, gP, nP, mom["mP"], mom["vP"]), (Q, gQ, nQ, mom["mQ"], mom["vQ"])):
            ref, mag = _opt_ref(opt, T, g, m, v, lr, s + 1)
            bound = 2 * U_RND * np.abs(ref) + OPT_ULPS * U_RND * mag
            err = np.abs(got.astype(np.float64) - ref)
            with np.errstate(divide="ignore", invalid="ignore"):
                r = np.where(err > 0, err / bound, 0.0)
            worst = max(worst, float(r.max()))
        assert ws_fixed_zero(run.ws)
    print(f"{opt}: worst error / bound {worst:.3g}")
    assert worst <= 1.0, worst


@pytest.mark.gpu
def test_det_reg2_vs_fp64_at_ml20m_shape():
    """reg_2 != 0 (the batch norms, the 2^-32 scalar sums): the fp64 bound of test_gpu_mf_step_fp64 and its LOSS_RTOL, two
    teacher-forced launches at the bench shape"""
    import test_gpu_mf_step_fp64 as mfs
    U, I, F, B = ML20M
    rng = np.random.default_rng(4)
    P0, Q0 = (rng.standard_normal((U, F)) * 0.01).astype(F32), (rng.standard_normal((I, F)) * 0.01).astype(F32)
    planes = ml20m_batches(2, seed=21)

    class DetStep(mfs.GpuStep):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            self.ws = self.ops.MFWorkspace(U, I, F, "sgd", "cuda", deterministic=True)

        def workspace_zero(self):
            return ws_fixed_zero(self.ws)

    st = DetStep(P0, Q0, planes, "sgd", 0.01)
    recs = [mfs.sgd_launch(st, s * B, B, B, 1, 0.01, 0.001, 0.001, tag=f"det-reg2-{s}") for s in range(2)]
    for r in recs:
        print({k: r[k] for k in ("tag", "ratio", "kappa_need", "loss_rel", "ws_zero")})
    assert all(r["ok"] for r in recs), recs


@pytest.mark.gpu
@pytest.mark.parametrize("how", ["loss", "table-sum", "in-range"])
def test_det_out_of_range_is_reported(how):
    """SL under deterministic=True.  loss: labels of 2^30, so one triple's loss is beyond the 2^62-unit value limit of the
    scalar sums.  table-sum: q_i = 0, p = 10 and label 1000 on one item, 1024 times: each contribution 2e4 is in range, their
    sum 2e7 is past the 2^23 range of a table element.  Both must raise the non-finite-loss ValueError and leave the tables
    alone; in-range (label 100, sum 2e6) must not."""
    torch, ops = _torch_ops()
    U, I, F, B = 64, 32, 8, 1024
    rng = np.random.default_rng(29)
    P0 = np.full((U, F), 10.0, F32) if how != "loss" else (rng.standard_normal((U, F)) * 0.1).astype(F32)
    Q0 = np.zeros((I, F), F32) if how != "loss" else (rng.standard_normal((I, F)) * 0.1).astype(F32)
    label = {"loss": 1 << 30, "table-sum": 1000, "in-range": 100}[how]
    planes = (rng.integers(U, size=B).astype(np.int32), np.zeros(B, np.int32), np.full(B, label, np.int32))
    run = DetRun(P0, Q0)
    if how == "in-range":
        loss = run.launch(planes, B, 1, 0.001, 0.0, 0.0, "SL")
        assert np.isfinite(loss).all()
        assert not np.array_equal(run.tables()[1], Q0)
        return
    with pytest.raises(ValueError, match="Nan or Infinity"):
        run.launch(planes, B, 1, 0.001, 0.0, 0.0, "SL")
    P, Q = run.tables()
    assert np.array_equal(P, P0) and np.array_equal(Q, Q0)


# ---------------------------------------------------------------- GPU: independence of the triple-to-thread map
TILE_CAPS = ["", "256", "1024"]      # "" = the default cap (512)
TILE_CASES = [("BPR", "sgd", 0.001, 0.0), ("BPR", "sgd", 0.001, 0.001), ("BPR", "adam", 0.001, 0.001),
              ("HL", "sgd", 0.001, 0.001), ("TL", "sgd", 0.001, 0.001), ("CL", "sgd", 0.001, 0.001),
              ("SL", "rmsprop", 0.001, 0.001)]


def tile_child(out):
    """every TILE_CASE at the bench shape, 2-step launch from the same seeded start -> npz of Q, the sha256 of P, losses"""
    U, I, F, B = ML20M
    res = {}
    for n, (loss, opt, r1, r2) in enumerate(TILE_CASES):
        rng = np.random.default_rng(100 + n)
        P0, Q0 = (rng.standard_normal((U, F)) * 0.1).astype(F32), (rng.standard_normal((I, F)) * 0.1).astype(F32)
        planes = ml20m_batches(2, loss, seed=31)
        run = DetRun(P0, Q0, opt)
        loss_v = run.launch(planes, B, 2, 0.01, r1, r2, loss)
        P, Q = run.tables()
        res[f"Q{n}"] = Q
        res[f"L{n}"] = loss_v
        res[f"P{n}"] = np.frombuffer(hashlib.sha256(P.tobytes()).digest(), np.uint8)
    np.savez(out, **res)


@pytest.mark.gpu
def test_det_result_does_not_depend_on_the_tile_size(tmp_path):
    outs = []
    for cap in TILE_CAPS:
        env = dict(os.environ)
        env.pop("DRB_TILE_CAP", None)
        if cap:
            env["DRB_TILE_CAP"] = cap
        out = str(tmp_path / f"tile{cap or 'default'}.npz")
        t0 = time.time()
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "tile", out], env=env, capture_output=True, text=True,
                           timeout=1200)
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
        print(f"tile cap {cap or 'default'}: {time.time() - t0:.1f} s")
        outs.append(np.load(out))
    bad = []
    for n, case in enumerate(TILE_CASES):
        for cap, o in zip(TILE_CAPS[1:], outs[1:]):
            a, b = outs[0], o
            dq = int((a[f"Q{n}"] != b[f"Q{n}"]).sum())
            same_p = np.array_equal(a[f"P{n}"], b[f"P{n}"])
            same_l = np.array_equal(a[f"L{n}"], b[f"L{n}"])
            print(case, f"cap {cap}: Q elements differing {dq}, P equal {same_p}, losses {a[f'L{n}']} / {b[f'L{n}']}")
            if dq or not same_p or not same_l:
                bad.append((case, cap, dq, same_p, same_l))
    assert not bad, bad


# ---------------------------------------------------------------- GPU: fused negatives, bit for bit
def _fused_launch(P0, Q0, bu, bi, row_ptr, col, seed, B, first, k, opt="sgd", reg=(0.001, 0.001)):
    torch, ops = _torch_ops()
    P, Q = _dev(P0), _dev(Q0)
    ws = ops.MFWorkspace(P0.shape[0], Q0.shape[0], P0.shape[1], opt, "cuda")
    neg = torch.full((len(bu),), -1, dtype=torch.int32, device="cuda")
    loss = ops.mf_bpr_train_steps_fused_neg(P, Q, ws, _dev(bu), _dev(bi), _dev(row_ptr), _dev(col), seed, B, first, k,
                                            ops.hyper(0.01, *reg, opt), neg_out=neg)
    torch.cuda.synchronize()
    return neg.cpu().numpy(), loss.cpu().numpy(), P, Q


@pytest.mark.gpu
def test_fused_negatives_bit_exact_ml20m():
    """the ML-20M CSR at the bench batch, a 3-step launch at first_step 2"""
    cu, ci, row_ptr, col = ml20m_positives()
    U, I, F, B = ML20M
    rng = np.random.default_rng(17)
    sel = rng.permutation(len(cu))[:5 * B]
    bu, bi = cu[sel].astype(np.int32), ci[sel].astype(np.int32)
    P0, Q0 = (rng.standard_normal((U, F)) * 0.01).astype(F32), (rng.standard_normal((I, F)) * 0.01).astype(F32)
    seed = 0x5DEECE66D
    neg, _, _, _ = _fused_launch(P0, Q0, bu, bi, row_ptr, col, seed, B, 2, 3)
    gt = np.arange(2 * B, 5 * B, dtype=np.uint64)
    want = draw_negatives(row_ptr, col, I, seed, bu[2 * B:], gt, gt // np.uint64(B))
    assert (neg[:2 * B] == -1).all()
    assert np.array_equal(neg[2 * B:], want), int((neg[2 * B:] != want).sum())


@pytest.mark.gpu
def test_fused_negatives_bit_exact_crafted_rows():
    """empty row, one missing item (middle, 0, I - 1), a hub row over 2^16, a seed above 2^32, 3 steps at first_step 2"""
    I, row_ptr, col = crafted_csr()
    U, F, B = len(row_ptr) - 1, 8, 4096
    rng = np.random.default_rng(19)
    n = 5 * B
    bu = np.concatenate([np.arange(5), rng.integers(U, size=n - 5)]).astype(np.int32)
    bu[rng.random(n) < 0.3] = 4                                   # the hub row
    bi = np.array([col[row_ptr[u] + rng.integers(max(1, row_ptr[u + 1] - row_ptr[u]))] if row_ptr[u + 1] > row_ptr[u] else 0
                   for u in bu], np.int32)
    P0, Q0 = (rng.standard_normal((U, F)) * 0.1).astype(F32), (rng.standard_normal((I, F)) * 0.1).astype(F32)
    seed = (0xA5 << 32) + 0x1234567
    neg, _, _, _ = _fused_launch(P0, Q0, bu, bi, row_ptr, col, seed, B, 2, 3)
    gt = np.arange(2 * B, 5 * B, dtype=np.uint64)
    u = bu[2 * B:]
    want = draw_negatives(row_ptr, col, I, seed, u, gt, gt // np.uint64(B))
    got = neg[2 * B:]
    assert np.array_equal(got, want), int((got != want).sum())
    assert (got[u == 1] == 31_337).all() and (got[u == 2] == 0).all() and (got[u == 3] == I - 1).all()
    assert got[u == 0].max() > I - I // 20


@pytest.mark.gpu
def test_fused_launch_vs_fp64_on_recorded_negatives():
    """one fused single-step launch checked with the fp64 bound of test_gpu_mf_step_fp64 on the negatives it drew"""
    import test_gpu_mf_step_fp64 as mfs
    rng = np.random.default_rng(23)
    U, I, F, B, nnz = 1200, 900, 64, 4096, 40_000
    cu = rng.integers(U, size=nnz).astype(np.int32)
    ci = np.minimum(I - 1, rng.zipf(1.2, size=nnz) - 1).astype(np.int32)
    key = np.unique(cu.astype(np.int64) * I + ci)
    row_ptr = np.searchsorted(key // I, np.arange(U + 1)).astype(np.int64)
    col = (key % I).astype(np.int32)
    sel = rng.integers(nnz, size=B)
    bu, bi = cu[sel], ci[sel]
    P0, Q0 = (rng.standard_normal((U, F)) * 0.1).astype(F32), (rng.standard_normal((I, F)) * 0.1).astype(F32)
    seed = 99

    class FusedStep:
        def __init__(self):
            self.P, self.Q, self.neg = P0.copy(), Q0.copy(), None

        def tables(self):
            return self.P.copy(), self.Q.copy()

        def batch(self, lo, n):
            return bu[lo:lo + n], bi[lo:lo + n], self.neg[lo:lo + n]

        def __call__(self, lo, n, batch, k, reg1, reg2, adam_step0=0):
            neg, loss, P, Q = _fused_launch(self.P, self.Q, bu, bi, row_ptr, col, seed, B, 0, 1, reg=(reg1, reg2))
            self.neg, self.P, self.Q = neg, P.cpu().numpy(), Q.cpu().numpy()
            return loss, None

        def workspace_zero(self):
            return True

    st = FusedStep()
    rec = mfs.sgd_launch(st, 0, B, B, 1, 0.01, 0.001, 0.001, tag="fused")
    print({k: rec[k] for k in ("ratio", "kappa_need", "loss_rel")})
    assert np.array_equal(st.neg, draw_negatives(row_ptr, col, I, seed, bu, np.arange(B, dtype=np.uint64), 0))
    assert rec["ok"], rec


if __name__ == "__main__":
    if sys.argv[1] == "tile":
        tile_child(sys.argv[2])
