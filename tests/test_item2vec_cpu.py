"""The numpy restatement of Item2Vec (oracle/i2v_oracle.py) against tests/golden/item2vec.npz, the reference's own runs."""
import hashlib

import numpy as np
import torch

from conftest import golden
from oracle import i2v_oracle as io


def _case(g, k):
    U, I, w, discard, seed = (int(v) for v in g[f"s{k}_meta"])
    users, items = g[f"s{k}_users"], g[f"s{k}_items"]
    ur = {}
    for u, i in zip(users.tolist(), items.tolist()):
        ur.setdefault(u, set()).add(i)
    for u, i in g[f"s{k}_extra_ur"].tolist():
        ur.setdefault(u, set()).add(i)
    return U, I, w, bool(discard), seed, users, items, ur


def _state():
    s = np.random.get_state()
    return np.concatenate([s[1].astype(np.int64), [int(s[2])]])


def _ml_train():
    """Config 1's ml-100k train rows (the item2vec fixture was generated on the same split) and train_ur, its sets filled in
    row order as get_ur fills them (so that list(ur[u]) has the reference's order)."""
    gs = golden("ml100k_sampler")
    cu, ci = gs["coo_u"].astype(np.int64), gs["coo_i"].astype(np.int64)
    ur = {}
    for u, i in zip(cu.tolist(), ci.tolist()):
        ur.setdefault(u, set()).add(i)
    return cu, ci, ur


def _ml_test_ur():
    gr = golden("ml100k_rank")
    off = np.concatenate([[0], np.cumsum(gr["gt_len"])])
    return {int(u): gr["gt_flat"][off[k]:off[k + 1]].tolist() for k, u in enumerate(gr["test_u"])}


def _ml_init(g):
    """The reference's initial tables: nn.Embedding(user_num), nn.Embedding(item_num), then N(0, 0.01) re-initialisation."""
    U, I, F, _, seed = (int(v) for v in g["ml_meta"][:5])
    torch.manual_seed(seed)
    P, Q = torch.empty(U, F).normal_(), torch.empty(I, F).normal_()
    torch.nn.init.normal_(P, 0.0, 0.01)
    torch.nn.init.normal_(Q, 0.0, 0.01)
    P, Q = P.numpy(), Q.numpy()
    assert hashlib.sha256(P.tobytes()).digest() == g["ml_P0_sha"].tobytes()
    assert hashlib.sha256(Q.tobytes()).digest() == g["ml_Q0_sha"].tobytes()
    return P, Q


def test_sampler_synthetic_cases():
    g = golden("item2vec")
    for k in range(int(g["n_synthetic"])):
        U, I, w, discard, seed, users, items, ur = _case(g, k)
        np.random.seed(seed)
        if discard:
            users, items = io.discard_rows(users, items, 0.5)
        rows = io.skipgram_rows(io.group_sequences(users, items), ur, I, w)
        assert np.array_equal(rows, g[f"s{k}_rows"].astype(np.int64)), k
        assert np.array_equal(_state(), g[f"s{k}_state"]), k


def test_sampler_ml100k_digest():
    g = golden("item2vec")
    U, I, F, w, seed = (int(v) for v in g["ml_meta"][:5])
    cu, ci, ur = _ml_train()
    np.random.seed(seed)
    rows = io.skipgram_rows(io.group_sequences(cu, ci), ur, I, w)
    assert rows.shape[0] == int(g["ml_meta"][6])
    assert hashlib.sha256(rows.tobytes()).digest() == g["ml_rows_sha"].tobytes()
    e = len(g["ml_rows_head"])
    assert np.array_equal(rows[:e], g["ml_rows_head"]) and np.array_equal(rows[-e:], g["ml_rows_tail"])
    assert np.array_equal(_state(), g["ml_state"])


def test_steps_ml100k():
    g = golden("item2vec")
    B, stride, lr = int(g["ml_meta"][5]), int(g["ml_meta"][7]), float(g["ml_lr"])
    rows = g["ml_rows_head"].astype(np.int64)
    _, Q0 = _ml_init(g)
    for opt in ("sgd", "adam"):
        Q = Q0.astype(np.float64)
        adam = (np.zeros_like(Q), np.zeros_like(Q))
        losses = [io.i2v_step(Q, rows[s * B:(s + 1) * B], lr, opt, adam, s + 1) for s in range(3)]
        assert np.allclose(losses, g[f"ml_{opt}_losses"], rtol=1e-5, atol=0), opt
        err = np.abs(Q[::stride] - g[f"ml_{opt}_Q3"])
        if opt == "sgd":
            assert err.max() <= 3e-6
        else:
            # Adam divides by sqrt(v) + eps: a slot whose gradient is ~0 in fp64 takes a step of any size up to lr in fp32
            # (m / sqrt(v) of rounding noise); the slots with a real gradient agree to 2e-5 of lr-sized steps
            moved = np.abs(adam[0][::stride]) > 1e-4 * np.abs(adam[0]).max()
            assert err[moved].max() <= 2e-5 * 3 and err.max() <= 3 * lr * 1.01


def test_user_embedding_and_rank():
    g = golden("item2vec")
    U, I, stride = int(g["ml_meta"][0]), int(g["ml_meta"][1]), int(g["ml_meta"][7])
    _, _, ur = _ml_train()
    Q = g["ml_fit_Q"]
    P0, _ = _ml_init(g)
    P64 = io.user_embedding(Q, ur, P0)
    want = g["ml_fit_P"]
    assert np.allclose(P64[::stride], want, rtol=1e-6, atol=1e-6 * np.abs(want).max())
    # the reference's own fp32 sums (Item2VecRecommender.py:58-61), then rank (:79-95) on its candidate sets: its lists, id for id
    Qt = torch.from_numpy(Q)
    Pt = torch.from_numpy(P0.copy())
    for u in ur:
        Pt[u] = Qt[torch.tensor(list(ur[u]))].sum(dim=0)
    assert np.array_equal(Pt.numpy()[::stride], want)
    np.random.set_state(("MT19937", g["ml_state"][:624].astype(np.uint32), int(g["ml_state"][624]), 0, 0.0))
    test_u, cands = io.build_candidates_set(_ml_test_ur(), ur, I, 1000)
    assert hashlib.sha256(cands.tobytes()).digest() == g["ml_cands_sha"].tobytes()
    us, cands = torch.tensor(test_u), torch.from_numpy(cands)
    scores = torch.bmm(Pt[us].unsqueeze(1), Qt[cands].transpose(1, 2)).squeeze()
    top = torch.gather(cands, 1, torch.argsort(scores, descending=True))[:, :50]
    assert np.array_equal(top.numpy(), g["ml_preds"].astype(np.int64))
