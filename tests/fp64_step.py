"""The float64 step check shared by test_gpu_graph_fp64.py, test_gpu_nfm_fm_fp64.py and test_gpu_neumf_bf16_fp64.py (a helper
module: pytest does not collect it).

One teacher-forced step.  Before every checked step the device's parameters and optimiser state (read from its workspace
through a mirror of the library's carve) are snapshotted; the model's float64 reference runs the same batch on that snapshot
and the device's post-step parameters are compared element-wise, so errors never compound.

Bound, per element e of every parameter tensor (u = 2^-24):

    SGD   |gpu - ref| <= 2 u |theta| + lr (KAPPA u N_e + P_e)

N_e is the sum of |contributions| along the chain, computed by running the same chain on absolute values, each operand
carrying its own fp32 noise forward.  P_e is the discrete part: a value whose noise interval (KAPPA u N + P) contains a bf16
rounding midpoint may round to its neighbour (the bf16 step goes to P and is carried through the downstream products); a gate
(relu, LeakyReLU, a hinge) whose input lies within its noise of the kink may go either way.  Every element that needs P_e
(error above the KAPPA-only bound) must have P_e > 0, and the flagged intermediates (those within their noise of a midpoint
or a kink) must stay under a ceiling fraction of all rounded / gated values.  The loss meets KAPPA u lossN + lossP.
Adam, Adagrad and RMSprop: the moments are read back and the update is evaluated across the gradient's noise interval
[g - e, g + e]; Adam's update (a + b g) / sqrt(c + d g^2) is not monotone, so 0 and its extremum g* = b c / (a d) are also
taken wherever they fall inside.  Under SGD elements with no contribution at all (N = P = 0) must stay bit-identical.

KAPPA is calibrated per model on the GPU and stated, with the measurements behind it, in each test module.  KAPPA_LADDER
feeds the "kappa needed" diagnostic of steps where no per-element KAPPA can be read off (Adam, bf16); it never changes a
verdict.

The references run on the CPU by default; the GPU tests run them in float64 on the GPU, which only makes them faster.
"""
import math

import numpy as np
import torch

U_RND = 2.0 ** -24
F64 = torch.float64
GAMMA = float(np.float32(1e-10))
KAPPA_LADDER = (0.125, 0.25, 0.5, 1, 1.5, 2, 3, 4, 6, 8, 12, 16, 24, 32, 48, 64)


# ---------------------------------------------------------------- noise-carrying primitives
def br(x):
    """bf16(fp32(x)) as a tensor of x's dtype (round to nearest even, from the fp32 bits; exactly representable in it)."""
    f = x.to(torch.float32).contiguous()
    b = f.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    r = (b + 0x7FFF + ((b >> 16) & 1)) & 0xFFFF0000
    r = torch.where(r >= 2 ** 31, r - 2 ** 32, r).to(torch.int32)
    return torch.where(torch.isnan(f), f, r.view(torch.float32)).to(x.dtype)


def flip(v, e):
    """the largest change of bf16(v) when v moves by at most e (0 unless [v - e, v + e] holds a rounding midpoint)"""
    r = br(v)
    return torch.maximum((br(v + e) - r).abs(), (br(v - e) - r).abs()).to(F64)


def _A(x):
    return x.abs().to(F64)


class Flags:
    """the rounded or gated intermediates of one step that may round / gate the other way (flag) of all of them (total), at
    the step's KAPPA (k)"""

    def __init__(self, k):
        self.k, self.flag, self.total = k, 0, 0

    def add(self, mask):
        self.flag += int(mask.sum()); self.total += mask.numel()

    def frac(self):
        return self.flag / max(1, self.total)


def rnd(v, vN, vP, fl, on=True):
    """a GEMM operand: bf16 (its possible midpoint flip in P, continuous noise dropped) or, off, fp32 as it is"""
    if not on:
        return v, vN, vP
    p = flip(v, fl.k * U_RND * vN + vP + U_RND * _A(v))
    fl.add(p > 0)
    return br(v), torch.zeros_like(vN), p


def mm(a, aN, aP, b, bN, bP, transpose_b):
    """a @ b(^T) with noise: (value, N, P)"""
    op = (lambda t: t.T) if transpose_b else (lambda t: t)
    v = a @ op(b)
    aA, bA = _A(a), _A(b)
    N = aA @ op(bA) + aN @ op(bA) + aA @ op(bN)
    P = aP @ op(bA) + aA @ op(bP)
    return v, N, P


# ---------------------------------------------------------------- optimiser mirrors
def adam_apply(th, g, m, v, lr, t):
    b1, b2, eps = np.float32(0.9), np.float32(0.999), 1e-8
    step_size = float(np.float32(lr / (1.0 - float(b1) ** t)))
    bc2 = float(np.float32(math.sqrt(1.0 - float(b2) ** t)))
    m2 = m + (g - m) * float(np.float32(1) - b1)
    v2 = v * float(b2) + float(np.float32(1) - b2) * g * g
    return th - step_size * (m2 / (torch.sqrt(v2) / bc2 + eps))


def adam_moments(g, m, v):
    b1, b2 = float(np.float32(1) - np.float32(0.9)), float(np.float32(1) - np.float32(0.999))
    return m + (g - m) * b1, v * float(np.float32(0.999)) + b2 * g * g


def opt_apply(th, g, st, lr, opt, t):
    """the update the device applies (float64 arithmetic on fp32 state): -> (theta, new state)"""
    if opt == "sgd":
        return th - lr * g, None
    if opt == "adam":
        m, v = st
        return adam_apply(th, g, m, v, lr, t), adam_moments(g, m, v)
    s = st[0]
    if opt == "adagrad":
        ss = s + g * g
        return th - lr * (g / (torch.sqrt(ss) + 1e-10)), (ss, None)
    sq = s * float(np.float32(0.99)) + float(np.float32(1) - np.float32(0.99)) * g * g
    return th - lr * (g / (torch.sqrt(sq) + 1e-8)), (sq, None)


def expect(th, g, N, P, lr, opt, kappa, mom=None, t=1):
    """-> (expected, half-width with KAPPA only, half-width with KAPPA and P) of one parameter tensor (float64)"""
    ek = kappa * U_RND * N
    if opt == "sgd":
        ex = th - lr * g
        base = 2 * U_RND * ex.abs()
        return ex, base + lr * ek, base + lr * (ek + P)
    f = lambda gg: opt_apply(th, gg, mom, lr, opt, t)[0]
    ex = f(g)
    # the fp32 update itself: about eight roundings on the step (moments, sqrt, scalings, division), the last one on theta
    base = 2 * U_RND * ex.abs() + 16 * U_RND * (ex - th).abs()
    inner = ()
    if opt == "adam":
        m, v = mom
        b1, b2 = float(np.float32(1) - np.float32(0.9)), float(np.float32(1) - np.float32(0.999))
        a_, c_ = m * (1 - b1), v * (1 - b2)
        inner = (torch.zeros_like(g), torch.nan_to_num(b1 * c_ / (a_ * b2), nan=0.0, posinf=0.0, neginf=0.0))
    out = []
    for e in (ek, ek + P):
        w = torch.zeros_like(g)
        for x in (g - e, g + e) + inner:
            w = torch.maximum(w, (f(torch.minimum(torch.maximum(x, g - e), g + e)) - ex).abs())
        out.append(base + w)
    return ex, out[0], out[1]


def compare(th, got, g, N, P, lr, opt, kappa, mom=None, t=1):
    """one parameter section (flat float64): worst error/bound and where, the elements above the KAPPA-only bound (widened;
    unflagged: those with P = 0, which fail), under SGD the KAPPA needed where P = 0 and the stray changes -> record"""
    ex, hk, hf = expect(th, g, N, P, lr, opt, kappa, mom, t)
    err = (got - ex).abs()
    ratio = torch.where(err > 0, err / hf, torch.zeros_like(err))
    wid = err > hk
    contrib = (N > 0) | (P > 0)
    rec = dict(ratio=float(ratio.max()) if ratio.numel() else 0.0, worst=int(ratio.argmax()) if ratio.numel() else -1,
               widened=int(wid.sum()), frac=float(wid.sum()) / max(1, int(contrib.sum())), unflagged=int((wid & (P == 0)).sum()),
               flagged=int((P > 0).sum()), kneed=float("nan"), kneed_at=-1, stray=0)
    if opt == "sgd":
        sel = (P == 0) & (N > 0)
        need = torch.where(sel, (err - 2 * U_RND * ex.abs()) / (lr * U_RND * N), torch.zeros_like(err))
        rec["kneed"] = float(need.max()) if need.numel() else 0.0
        rec["kneed_at"] = int(need.argmax()) if need.numel() else -1
        rec["stray"] = int(((got != th) & ~contrib).sum())
    rec["ok"] = bool(rec["ratio"] <= 1 and rec["unflagged"] == 0 and rec["stray"] == 0)
    return rec


# ---------------------------------------------------------------- workspace carve mirrors
def carve(parts):
    """the library's carve of a workspace: each part at the next 256-byte boundary -> ({name: (offset, bytes)}, total)"""
    out, off = {}, 0
    for name, nb in parts:
        out[name] = (off, nb)
        off += (nb + 255) // 256 * 256
    return out, off


def views(buf, layout, dtypes):
    """{name: the part's bytes of buf viewed as dtypes[name]} for every part named in dtypes"""
    return {k: buf[layout[k][0]:layout[k][0] + layout[k][1]].view(dt) for k, dt in dtypes.items()}


def device_tensor(a, device="cuda"):
    return (a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a))).to(device)


# ---------------------------------------------------------------- steppers
class Stepper:
    """What checked_step drives: the device or its CPU stand-in, both holding
    t: {name: fp32 tensor} (the parameters, plus state the model's checks read), planes: (bu, bi, bj),
    mom: {name: (m, v or None)} (workspace views on the device, float64 on the CPU; None under SGD), opt, lr, reg.
    A model supplies
    reference(pre, idx, kappa, **step) -> dict(g, N, P: {parameter name: float64}, loss, lossN, lossP, flagged),
    run(lo, n, batch, k, adam_step0, apply, first_step, **step) -> the step losses (the device's op call),
    sections() -> [(label, parameter name, lo, hi, row width)]: the flat slices compared separately,
    and may add model-specific exact checks (checks) and an accumulator check (clean)."""
    device = "cpu"
    kappa = phi_max = None
    td = 0
    ladder = True               # the KAPPA_LADDER diagnostic on Adam and bf16 steps
    ref_uses_kappa = True       # False: the reference's N and P do not depend on KAPPA (the ladder reuses one result)

    def _sync(self):
        if self.device != "cpu":
            torch.cuda.synchronize(self.device)

    def snapshot(self):
        self._sync()
        return {k: v.clone() for k, v in self.t.items()}

    def batch(self, lo, n):
        return tuple(p[lo:lo + n].long() for p in self.planes)

    def moments(self):
        if self.opt == "sgd":
            return None
        self._sync()
        return {k: tuple(None if x is None else x.to(F64).clone() for x in mv) for k, mv in self.mom.items()}

    def clean(self):
        """the gradient accumulators and row counters are zero"""
        return True

    def checks(self, pre, post, res, apply):
        """model-specific exact checks of one step -> {name: bool, or a ratio that must be <= 1}"""
        return {}


class StandIn(Stepper):
    """CPU stand-in of the device: the model's reference in float32 (optionally with defects) plays the step
    (stand_in_ref(idx, **step) -> reference result), the update is applied in fp32 through opt_apply"""

    def __init__(self, tabs, planes, opt, lr, reg, defects=()):
        self.t = {k: torch.from_numpy(np.array(v, np.float32)) for k, v in tabs.items()}
        self.planes = tuple(torch.from_numpy(np.asarray(p, np.int64)) for p in planes)
        self.opt, self.lr, self.reg, self.defects = opt, lr, reg, defects
        self.mom = {k: (torch.zeros(v.shape, dtype=F64), torch.zeros(v.shape, dtype=F64) if opt == "adam" else None)
                    for k, v in self.t.items()}

    def stand_in_ref(self, idx, **step):
        return self.reference(self.t, idx, self.kappa, torch.float32, self.defects, **step)

    def run(self, lo, n, batch, k, adam_step0=0, apply=True, first_step=0, **step):
        assert k == 1 and first_step == 0
        r = self.stand_in_ref(self.batch(lo, n), **step)
        if apply:
            for key, g in r["g"].items():
                T = self.t[key]
                gq = g.reshape(T.shape).to(torch.float32).to(F64)
                new, st = opt_apply(T.to(F64), gq, self.mom[key], self.lr, self.opt, adam_step0 + 1)
                T.copy_(new.to(torch.float32))
                if st is not None:
                    self.mom[key] = st
        return np.array([np.float32(r["loss"])], np.float64)


# ---------------------------------------------------------------- one teacher-forced step
def loss_ratio(lerr, res, kappa):
    lb = kappa * U_RND * res["lossN"] + res["lossP"]
    return lerr / lb if lb > 0 else float(lerr > 0)


def _judge(st, pre, post, mom, res, kappa, t):
    out = {}
    for label, key, lo, hi, w in st.sections():
        flat = lambda x: x.to(F64).reshape(-1)[lo:hi]
        mv = None if mom is None else tuple(None if x is None else flat(x) for x in mom[key])
        c = compare(flat(pre[key]), flat(post[key]), *(flat(res[x][key]) for x in ("g", "N", "P")), st.lr, st.opt, kappa, mv, t)
        at = lambda k: f"{label}[{k // w}, {k % w}]" if w > 1 else f"{label}[{k}]"
        c["worst_at"], c["kneed_at"] = at(c["worst"]), at(c["kneed_at"]) if st.opt == "sgd" else ""
        out[label] = c
    return out


def _passes(checks):
    return all(v <= 1 if isinstance(v, float) else bool(v) for v in checks.values())


def checked_step(st, lo, nb, batch, tag, adam_step0=0, apply=True, ref_device="cpu", with_res=False, ladder=None, **step):
    """one teacher-forced step of nb rows from row lo against st.reference -> record (and the reference result if with_res).
    step: per-step inputs (dropout masks) passed to both st.reference and st.run.  ladder (default: st.ladder on Adam,
    Adagrad, RMSprop and bf16 steps): also the smallest KAPPA of KAPPA_LADDER at which the step passes ("kneed")"""
    pre = st.snapshot()
    mom = st.moments()
    idx = tuple(x.to(ref_device) for x in st.batch(lo, nb))
    pre = {k: v.to(ref_device) for k, v in pre.items()}
    res = st.reference(pre, idx, st.kappa, **step)
    loss = st.run(lo, nb, batch, 1, adam_step0=adam_step0, apply=apply, **step)
    post = {k: v.to(ref_device) for k, v in st.snapshot().items()}
    lerr = abs(float(loss[0]) - res["loss"])
    rec = dict(tag=tag, nb=nb, loss=float(loss[0]), loss_ref=res["loss"], loss_ratio=loss_ratio(lerr, res, st.kappa),
               loss_rel=lerr / max(abs(res["loss"]), 1e-30), flagged=res["flagged"], tensors={},
               checks=st.checks(pre, post, res, apply))
    if not apply:
        mom2 = st.moments()
        rec["unchanged"] = (all(bool(torch.equal(pre[k], post[k])) for k in res["g"]) and
                            (mom is None or all(bool(torch.equal(a, b)) for k in mom for a, b in zip(mom[k], mom2[k])
                                                if a is not None)))
        rec["ok"] = bool(rec["unchanged"] and rec["loss_ratio"] <= 1 and _passes(rec["checks"]))
        return (rec, res) if with_res else rec
    mom = None if mom is None else {k: tuple(None if x is None else x.to(ref_device) for x in mv) for k, mv in mom.items()}
    t = rec["tensors"] = _judge(st, pre, post, mom, res, st.kappa, adam_step0 + 1)
    worst = max(t.values(), key=lambda c: c["ratio"])
    rec["ratio"], rec["worst_at"], rec["frac"] = worst["ratio"], worst["worst_at"], max(c["frac"] for c in t.values())
    kn = [(c["kneed"], c["kneed_at"]) for c in t.values() if not math.isnan(c["kneed"])]
    rec["kneed"], rec["kneed_at"] = max(kn) if kn else (float("nan"), "")
    rec["ok"] = bool(all(c["ok"] for c in t.values()) and rec["loss_ratio"] <= 1 and rec["flagged"] <= st.phi_max
                     and _passes(rec["checks"]))
    if ladder is None:
        ladder = st.ladder and (st.opt != "sgd" or st.td == 1)
    if ladder:
        rec["kneed"], rec["kneed_at"] = float("inf"), "-"
        for k in KAPPA_LADDER:
            rk = st.reference(pre, idx, k, **step) if st.ref_uses_kappa else res
            if all(c["ok"] for c in _judge(st, pre, post, mom, rk, k, adam_step0 + 1).values()) and loss_ratio(lerr, rk, k) <= 1:
                rec["kneed"], rec["kneed_at"], rec["flagged_at_kneed"] = k, "ladder", rk["flagged"]
                break
    return (rec, res) if with_res else rec


def launch_vs_singles(multi, single, n, batch, k, first_step=0, states=True, ref_device="cuda", step_of=None, **step):
    """one k-step launch of `multi` (rows [0, n), steps first_step ..) against k single launches of `single` from the same
    start, each checked against the reference (with the per-step inputs `step`, or step_of(s) for step s when given: each
    step's own dropout masks) -> the singles' records and one record of the launch: each launch step's loss
    within the bound of the single's reference, and (states) the launch's end state within the singles' end state plus twice
    the sum of their per-step half-widths 2 u |theta| + lr (KAPPA u N + P) (both runs lie within the bound of the same
    exact trajectory), every element of every parameter tensor"""
    losses = multi.run(0, n, batch, k, first_step=first_step)
    recs, acc, lrat = [], {}, []
    for s in range(first_step, first_step + k):
        pre = single.snapshot()
        r, res = checked_step(single, s * batch, min(batch, n - s * batch), batch, f"single {s}", adam_step0=s,
                              ref_device=ref_device, with_res=True, **(step if step_of is None else step_of(s)))
        recs.append(r)
        lrat.append(abs(float(losses[s - first_step]) - res["loss"]) / (single.kappa * U_RND * res["lossN"] + res["lossP"]))
        for key in res["g"]:
            hw = (2 * U_RND * pre[key].to(ref_device).to(F64).abs().reshape(-1)
                  + single.lr * (single.kappa * U_RND * res["N"][key].reshape(-1) + res["P"][key].reshape(-1)))
            acc[key] = hw if key not in acc else acc[key] + hw
    tens = {}
    if states:
        ea, eb = multi.snapshot(), single.snapshot()
        for key, h in acc.items():
            d = (ea[key].to(ref_device).to(F64) - eb[key].to(ref_device).to(F64)).abs().reshape(-1)
            rt = float(torch.where(d > 0, d / (2 * h), torch.zeros_like(d)).max())      # d > 0 where h == 0: inf
            tens[key] = dict(ratio=rt, ok=rt <= 1)
    worst = max((c["ratio"] for c in tens.values()), default=0.0)
    clean = multi.clean()
    recs.append(dict(tag=f"{k}-step launch vs {k} singles", nb=n, loss=float(losses[-1]), loss_ref=float("nan"),
                     loss_ratio=max(lrat), ratio=worst, kneed=float("nan"), tensors=tens, checks=dict(clean=clean),
                     ok=bool(worst <= 1 and max(lrat) <= 1 and clean)))
    return recs


def summary(rec):
    bad = {k: v for k, v in rec.get("tensors", {}).items() if not v["ok"]}
    checks = "".join(f" {k}={v:.3g}" if isinstance(v, float) else f" {k}={v}" for k, v in rec.get("checks", {}).items())
    return (f"{rec['tag']:36s} nb={rec['nb']:>8d} ratio={rec.get('ratio', 0):.3g} at {rec.get('worst_at', '-')} "
            f"kneed={rec.get('kneed', float('nan')):.3g} at {rec.get('kneed_at', '-')} flagged={rec.get('flagged', 0):.3g} "
            f"(at kneed {rec.get('flagged_at_kneed', float('nan')):.3g}) phi_frac={rec.get('frac', 0):.2g} "
            f"loss_ratio={rec['loss_ratio']:.3g} loss_rel={rec.get('loss_rel', 0):.2g}{checks}"
            + ("" if rec["ok"] else f"  FAIL {bad}"))


def report(key, recs):
    """print every record and the case's worst numbers, then assert every record passed"""
    checked = [r for r in recs if "ratio" in r]
    worst = max((r["ratio"] for r in checked), default=0.0)
    kn = max((r["kneed"] for r in checked if not math.isnan(r.get("kneed", float("nan")))), default=float("nan"))
    fl = max((r.get("flagged", 0.0) for r in recs), default=0.0)
    fr = max((r.get("frac", 0.0) for r in checked), default=0.0)
    for r in recs:
        print("  " + summary(r))
    print(f"[{key}] worst error/bound {worst:.3g}, largest kappa needed {kn:.3g}, flagged fraction {fl:.3g}, "
          f"largest Phi-widened fraction {fr:.2g}")
    for r in recs:
        assert r["ok"], summary(r)
