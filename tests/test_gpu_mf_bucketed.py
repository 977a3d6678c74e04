"""The user-bucketed mode of the lean MF step kernel against the general instantiation.

Each side runs in a child process, because the instantiation is chosen once per process: DRB_UBUCKET=1 forces the bucketed mode
(once it has passed its on-device check), DRB_NO_LEAN=1 keeps the general kernel.  Same seeded problems, same steps; tolerances are
the on-device selection's (losses 1e-5 relative, tables 1e-5 absolute; under Adam a few elements whose gradient is rounding noise
may move by up to 2 lr either way).
"""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CHILD = r"""
import ctypes
import sys
import numpy as np
import torch
sys.path.insert(0, sys.argv[1])
from daisyrec_b200 import _lib as L, ops
out, F, opt, U, I, B, n, hot, lr = sys.argv[2], int(sys.argv[3]), sys.argv[4], *map(int, sys.argv[5:10]), float(sys.argv[10])
rng = np.random.default_rng(F * 7 + U)
u = rng.integers(U, size=n).astype(np.int32)
if hot:
    u[np.arange(n) % 5 < 2] = 7                     # user 7: 40 % of every step, more triples than an index tile holds
    empty = (u >= 32) & (u < 48)                    # users 32..47 (one bucket at the smallest bucket width) never occur
    u[empty] += 16
i = (rng.random(n) ** 2 * I).astype(np.int32)
j = rng.integers(I, size=n).astype(np.int32)
P = torch.from_numpy((rng.standard_normal((U, F)) * 0.1).astype(np.float32)).cuda()
Q = torch.from_numpy((rng.standard_normal((I, F)) * 0.1).astype(np.float32)).cuda()
bu, bi, bj = (torch.from_numpy(x).cuda() for x in (u, i, j))
ws = ops.MFWorkspace(U, I, F, opt, "cuda")
hp = ops.hyper(lr, 0.001, 0.001, opt=opt)
K = (n + B - 1) // B
losses, modes, forms = [], [], []                    # modes: the instantiation each launch ran (2 = user-bucketed)
for first, k in ((0, 2), (2, K - 2)):
    losses.append(ops.mf_bpr_train_steps(P, Q, ws, bu, bi, bj, B, first, k, hp, adam_step0=first).cpu().numpy())
    modes.append(L.lib().drb_mf_last_step_mode())
    forms.append(L.lib().drb_mf_last_step_staged())   # 1: staged SGD form
torch.cuda.synchronize()
o = (ctypes.c_int64 * 8)()
L.check(L.lib().drb_mf_workspace_layout(U, I, F, L.OPT_KIND[opt], o))
buf = ws.buf
acc = [buf[o[6]:o[6] + 4 * U * F], buf[o[2]:o[2] + o[3]], buf[o[7]:o[7] + 4 * U], buf[o[4]:o[4] + o[5]]]
np.savez(out, P=P.cpu().numpy(), Q=Q.cpu().numpy(), loss=np.concatenate(losses),
         variant=L.lib().drb_mf_step_variant(F, U + I, None, None), modes=np.array(modes), forms=np.array(forms),
         acc_nonzero=sum(int(a.count_nonzero()) for a in acc))
"""


def run_child(tmp_path, tag, env_extra, args):
    out = str(tmp_path / f"{tag}.npz")
    env = dict(os.environ)
    env.pop("DRB_UBUCKET", None)
    env.pop("DRB_NO_LEAN", None)
    env.update(env_extra)
    r = subprocess.run([sys.executable, "-c", CHILD, ROOT, out] + [str(a) for a in args], env=env, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    return np.load(out)


# F, optimiser, U, I, batch, triples, hot user + empty bucket, lr (0.01 with a hot user: its large item sums carry fp32 noise of
# the general kernel itself near the 1e-5 tolerance at 0.05)
CASES = [
    pytest.param(64, "sgd", 3000, 500, 8192, 4 * 8192 + 3000, 0, 0.05, id="f64-sgd-ragged"),
    pytest.param(64, "adam", 3000, 500, 8192, 4 * 8192 + 3000, 0, 0.01, id="f64-adam-ragged"),
    pytest.param(64, "sgd", 20000, 2000, 1024, 5 * 1024, 0, 0.05, id="f64-sgd-claim-mode"),
    pytest.param(64, "sgd", 3001, 400, 4096, 3 * 4096, 1, 0.01, id="f64-sgd-hot-user-empty-bucket"),
    pytest.param(64, "adam", 3001, 400, 4096, 3 * 4096, 1, 0.01, id="f64-adam-hot-user-empty-bucket"),
    pytest.param(32, "sgd", 5000, 700, 8192, 3 * 8192 + 100, 1, 0.01, id="f32-sgd"),
    pytest.param(32, "adam", 5000, 700, 8192, 3 * 8192 + 100, 0, 0.01, id="f32-adam"),
    pytest.param(128, "sgd", 3000, 500, 8192, 3 * 8192, 1, 0.01, id="f128-sgd"),
    pytest.param(128, "adam", 3000, 500, 8192, 3 * 8192, 0, 0.01, id="f128-adam"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("F,opt,U,I,B,n,hot,lr", CASES)
def test_bucketed_matches_general(tmp_path, F, opt, U, I, B, n, hot, lr):
    args = (F, opt, U, I, B, n, hot, lr)
    ref = run_child(tmp_path, "general", {"DRB_NO_LEAN": "1"}, args)
    got = run_child(tmp_path, "bucketed", {"DRB_UBUCKET": "1"}, args)
    assert int(ref["variant"]) == 0 and list(ref["modes"]) == [0, 0]
    # the bucketed mode exists for the 8-lane x 1 | 2 chunk geometries (F = 32, 64); F = 128 keeps the plain lean kernel.  Both
    # launches of the child must have run it, not only the selection have chosen it.
    assert (int(got["variant"]) == 2) == (F in (32, 64))
    if F in (32, 64):
        assert list(got["modes"]) == [2, 2], got["modes"]
    else:
        assert 2 not in list(got["modes"]), got["modes"]
    # at these widths (16 users per bucket) the bucketed mode stages its user rows under SGD, and keeps the
    # accumulate-then-sweep user side under Adam
    staged = int(F in (32, 64) and opt == "sgd")
    assert list(got["forms"]) == [staged, staged] and list(ref["forms"]) == [0, 0], got["forms"]
    np.testing.assert_allclose(got["loss"], ref["loss"], rtol=1e-5)
    assert np.all(ref["loss"] > 0)
    for t in ("P", "Q"):
        d = np.abs(got[t] - ref[t])
        bad = d > 1e-5
        if opt == "adam":
            assert bad.sum() <= 4 and d.max() <= 2 * lr + 1e-6, (t, int(bad.sum()), float(d.max()))
        else:
            assert not bad.any(), (t, int(bad.sum()), float(d.max()))
    # workspace rule: gradient accumulators and row counters are all zero between launches
    assert int(got["acc_nonzero"]) == 0 and int(ref["acc_nonzero"]) == 0
