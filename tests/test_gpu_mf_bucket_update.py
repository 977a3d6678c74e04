"""The user-bucketed MF step under SGD, which stages each bucket's user rows in shared memory and updates them when the bucket
completes, against the general instantiation.

Each side runs in one child process for all cases, because the instantiation is chosen once per process: DRB_UBUCKET=1 forces
the bucketed mode (once it has passed its on-device check), DRB_NO_LEAN=1 keeps the general kernel.  Every case runs its steps
as two launches, so the per-launch norm cache of the bucketed side is built twice; one case rescales the user table between
them.  Tolerances are the on-device selection's: losses 1e-5 relative at every step, tables 1e-5 absolute.
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
for name, (F, U, I, B, n, hot, lr, reg, halve) in cases.items():
    rng = np.random.default_rng(F * 7 + U)
    u = rng.integers(U, size=n).astype(np.int32)
    if hot:
        u[np.arange(n) % 5 < 2] = 7                 # user 7: 40 % of every step, more triples than an index tile holds
        empty = (u >= 32) & (u < 48)                # users 32..47 (one bucket at the smallest bucket width) never occur
        u[empty] += 16
    i = (rng.random(n) ** 2 * I).astype(np.int32)
    j = rng.integers(I, size=n).astype(np.int32)
    P = torch.from_numpy((rng.standard_normal((U, F)) * 0.1).astype(np.float32)).cuda()
    Q = torch.from_numpy((rng.standard_normal((I, F)) * 0.1).astype(np.float32)).cuda()
    bu, bi, bj = (torch.from_numpy(x).cuda() for x in (u, i, j))
    ws = ops.MFWorkspace(U, I, F, "sgd", "cuda")
    hp = ops.hyper(lr, reg, reg, opt="sgd")
    K = (n + B - 1) // B
    o = (ctypes.c_int64 * 8)()
    L.check(L.lib().drb_mf_workspace_layout(U, I, F, L.OPT_KIND["sgd"], o))
    buf = ws.buf
    losses, modes, forms, nonzero = [], [], [], []
    for first, k in ((0, 2), (2, K - 2)):
        if first and halve:
            P.mul_(0.5)                             # the user norms the first launch cached are stale now
        losses.append(ops.mf_bpr_train_steps(P, Q, ws, bu, bi, bj, B, first, k, hp).cpu().numpy())
        modes.append(L.lib().drb_mf_last_step_mode())
        forms.append(L.lib().drb_mf_last_step_staged())
        torch.cuda.synchronize()
        # gP, gQ, cntU, cntI: zero between launches
        acc = [buf[o[6]:o[6] + 4 * U * F], buf[o[2]:o[2] + o[3]], buf[o[7]:o[7] + 4 * U], buf[o[4]:o[4] + o[5]]]
        nonzero.append(sum(int(a.count_nonzero()) for a in acc))
    np.savez(f"{outdir}/{name}.npz", P=P.cpu().numpy(), Q=Q.cpu().numpy(), loss=np.concatenate(losses), modes=np.array(modes),
             forms=np.array(forms), nonzero=np.array(nonzero))
"""

# name: F, U, I, batch, triples, hot user + empty bucket, lr, reg_1 = reg_2, halve P between the launches.  lr 0.01 with a hot
# user: its large item sums carry fp32 noise of the general kernel itself near the 1e-5 tolerance at 0.05.
CASES = {
    "f64": (64, 3000, 500, 8192, 4 * 8192 + 3000, 0, 0.05, 0.001, 0),            # ragged last step
    "f32": (32, 5000, 700, 8192, 3 * 8192 + 100, 0, 0.05, 0.001, 0),
    "f64-hot-user-empty-bucket": (64, 3001, 400, 4096, 3 * 4096, 1, 0.01, 0.001, 0),   # U = 187 x 16 + 9: partial last bucket
    "f32-hot-user-empty-bucket": (32, 5001, 700, 4096, 3 * 4096, 1, 0.01, 0.001, 0),
    "f64-claim-mode": (64, 20000, 2000, 1024, 5 * 1024, 0, 0.05, 0.001, 0),      # 3 B < (U + I) / 4: claim-mode phase 2
    "f32-claim-mode": (32, 20000, 2000, 1024, 5 * 1024, 0, 0.05, 0.001, 0),
    "f64-rescaled-between-launches": (64, 3000, 500, 8192, 4 * 8192, 0, 0.05, 0.001, 1),
    "f64-no-regulariser": (64, 3000, 500, 8192, 4 * 8192, 0, 0.05, 0.0, 0),     # no norm cache: the update without norms
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


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_bucket_update_matches_general(tmp_path_factory, name):
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
    # the bucketed side never writes gP / cntU, the general one clears what it wrote: all accumulators zero after each launch
    assert list(got["nonzero"]) == [0, 0] and list(ref["nonzero"]) == [0, 0]
