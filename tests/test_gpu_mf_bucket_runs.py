"""The user-bucketed MF step's per-tile user sort against the general instantiation.

Under the bucketed mode each index tile of a bucket is counting-sorted by user, and each lane group sums the user gradient of
its slice of the sorted tile in registers, one run of a user at a time: a run that lies inside one group's slice is added to
the bucket's shared accumulator with plain loads and stores, a run that crosses a slice boundary with shared-memory atomics.
Under SGD the item rows' regulariser is added once per occurrence in phase 1, and no item counter is written.  The cases put
runs at every boundary that logic has:
- a bucket of three tiles in which one user's run crosses both tile boundaries (and many slice boundaries);
- tiles that hold a single user (every other user of the bucket is absent);
- runs of length 1 (no user twice in a step);
- a ragged last step; F = 32 and 64; no regulariser.

Each side runs in one child process for all cases, because the instantiation is chosen once per process: DRB_UBUCKET=1 forces
the bucketed mode (once it has passed its on-device check), DRB_NO_LEAN=1 keeps the general kernel.  Tolerances are the
on-device selection's: losses 1e-5 relative at every step, tables 1e-5 absolute.  After each launch every accumulator (gP, gQ,
cntU, cntI) must be zero again.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CHILD = r"""
import ctypes
import json
import sys
import numpy as np
import torch
sys.path.insert(0, sys.argv[1])
from daisyrec_b200 import _lib as L, ops
outdir, cases = sys.argv[2], json.loads(sys.argv[3])
for name, (F, U, I, B, n, kind, lr, reg, opt) in cases.items():
    rng = np.random.default_rng(F * 11 + U + len(name))
    u = rng.integers(U, size=n).astype(np.int32)
    k = np.arange(n)
    if kind in ("hot", "single"):
        u[k % 10 < 3] = 7                           # user 7: 30 % of every step, its bucket (users 0..15) spans three tiles
        if kind == "single":
            other = (u < 16) & (u != 7)             # ... and holds no other user: its tiles are one run each
            u[other] += 16
    elif kind == "distinct":
        u = ((k % B) * 7919 % U).astype(np.int32)   # B <= U and 7919 prime to U: no user twice in a step
    i = (rng.random(n) ** 2 * I).astype(np.int32)
    j = rng.integers(I, size=n).astype(np.int32)
    P = torch.from_numpy((rng.standard_normal((U, F)) * 0.1).astype(np.float32)).cuda()
    Q = torch.from_numpy((rng.standard_normal((I, F)) * 0.1).astype(np.float32)).cuda()
    bu, bi, bj = (torch.from_numpy(x).cuda() for x in (u, i, j))
    ws = ops.MFWorkspace(U, I, F, opt, "cuda")
    hp = ops.hyper(lr, reg, reg, opt=opt)
    K = (n + B - 1) // B
    o = (ctypes.c_int64 * 8)()
    L.check(L.lib().drb_mf_workspace_layout(U, I, F, L.OPT_KIND[opt], o))
    buf = ws.buf
    losses, modes, forms, nonzero = [], [], [], []
    for first, cnt in ((0, 2), (2, K - 2)):
        losses.append(ops.mf_bpr_train_steps(P, Q, ws, bu, bi, bj, B, first, cnt, hp).cpu().numpy())
        modes.append(L.lib().drb_mf_last_step_mode())
        forms.append(L.lib().drb_mf_last_step_staged())
        torch.cuda.synchronize()
        # gP, gQ, cntU, cntI: zero between launches
        acc = [buf[o[6]:o[6] + 4 * U * F], buf[o[2]:o[2] + o[3]], buf[o[7]:o[7] + 4 * U], buf[o[4]:o[4] + o[5]]]
        nonzero.append(sum(int(a.count_nonzero()) for a in acc))
    np.savez(f"{outdir}/{name}.npz", P=P.cpu().numpy(), Q=Q.cpu().numpy(), loss=np.concatenate(losses), modes=np.array(modes),
             forms=np.array(forms), nonzero=np.array(nonzero))
"""

# name: F, U, I, batch, triples, user pattern, lr, reg_1 = reg_2, optimiser.  lr 0.01 with a hot user: its large item sums carry
# fp32 noise of the general kernel itself near the 1e-5 tolerance at 0.05.
CASES = {
    "f64-run-across-three-tiles": (64, 3000, 500, 8192, 4 * 8192, "hot", 0.01, 0.001, "sgd"),
    "f32-run-across-three-tiles": (32, 5000, 700, 8192, 4 * 8192, "hot", 0.01, 0.001, "sgd"),
    "f64-single-user-tiles": (64, 3000, 500, 8192, 4 * 8192, "single", 0.01, 0.001, "sgd"),
    "f32-single-user-tiles": (32, 5000, 700, 8192, 4 * 8192, "single", 0.01, 0.001, "sgd"),
    "f64-runs-of-one": (64, 20000, 2000, 8192, 4 * 8192, "distinct", 0.05, 0.001, "sgd"),
    "f32-runs-of-one": (32, 20000, 2000, 8192, 4 * 8192, "distinct", 0.05, 0.001, "sgd"),
    "f64-ragged-last-step": (64, 3000, 500, 8192, 4 * 8192 + 1000, "uniform", 0.05, 0.001, "sgd"),
    "f32-ragged-last-step": (32, 5000, 700, 8192, 3 * 8192 + 77, "uniform", 0.05, 0.001, "sgd"),
    "f64-no-regulariser": (64, 3000, 500, 8192, 4 * 8192, "hot", 0.01, 0.0, "sgd"),
    "f32-no-regulariser": (32, 20000, 2000, 8192, 4 * 8192, "distinct", 0.05, 0.0, "sgd"),
}

_OUT = {}


def _children(tmp_path_factory):
    if not _OUT:
        for tag, env_extra in (("general", {"DRB_NO_LEAN": "1"}), ("bucketed", {"DRB_UBUCKET": "1"})):
            out = tmp_path_factory.mktemp(tag)
            env = dict(os.environ)
            env.pop("DRB_UBUCKET", None)
            env.pop("DRB_NO_LEAN", None)
            env.update(env_extra)
            r = subprocess.run([sys.executable, "-c", CHILD, ROOT, str(out), json.dumps(CASES)], env=env, capture_output=True,
                               text=True, timeout=900)
            assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
            _OUT[tag] = out
    return _OUT


def test_cases_cover_the_sort_boundaries():
    """CPU: the hot cases put more than two and at most three index tiles (1 024 records) of the hot user's bucket in a step,
    and the runs-of-one cases never repeat a user within a step"""
    for name, (F, U, I, B, n, kind, lr, reg, opt) in CASES.items():
        k = np.arange(B)
        if kind in ("hot", "single"):
            hot = int((k % 10 < 3).sum())
            assert 2048 < hot <= 3 * 1024 - 16, name
        if kind == "distinct":
            assert B <= U and np.unique(k * 7919 % U).size == B, name


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_bucket_runs_match_general(tmp_path_factory, name):
    out = _children(tmp_path_factory)
    ref = np.load(out["general"] / f"{name}.npz")
    got = np.load(out["bucketed"] / f"{name}.npz")
    assert list(ref["modes"]) == [0, 0]
    assert list(got["modes"]) == [2, 2], got["modes"]       # both launches ran the bucketed mode
    assert list(got["forms"]) == [1, 1] and list(ref["forms"]) == [0, 0], got["forms"]   # in its staged SGD form
    assert np.all(ref["loss"] > 0)
    np.testing.assert_allclose(got["loss"], ref["loss"], rtol=1e-5)
    for t in ("P", "Q"):
        d = np.abs(got[t] - ref[t])
        assert not (d > 1e-5).any(), (t, int((d > 1e-5).sum()), float(d.max()))
    assert list(got["nonzero"]) == [0, 0] and list(ref["nonzero"]) == [0, 0]
