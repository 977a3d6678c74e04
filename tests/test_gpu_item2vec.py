"""Item2Vec on the GPU path: the skip-gram sampler, the tied-table step and the drop-in class against the reference's runs
(tests/golden/item2vec.npz) and the numpy restatement (oracle/i2v_oracle.py)."""
import hashlib
import logging

import numpy as np
import pandas as pd
import pytest
import torch

from conftest import golden
from oracle import i2v_oracle as io

pytestmark = pytest.mark.gpu


def _config(**kw):
    cfg = dict(gpu='0', seed=2022, topk=50, cand_num=1000, batch_size=256, init_method='default', optimizer='default',
               early_stop=False, UID_NAME='user', IID_NAME='item', INTER_NAME='rating', TID_NAME='timestamp', factors=32,
               epochs=1, lr=0.001, rho=0.5, context_window=2, loss_type='BPR', logger=logging.getLogger('t'), progress=False)
    cfg.update(kw)
    return cfg


def _df(users, items):
    return pd.DataFrame({"user": np.asarray(users, np.int64), "item": np.asarray(items, np.int64), "rating": 1.0,
                         "timestamp": np.arange(len(users))})


def _state():
    s = np.random.get_state()
    return np.concatenate([s[1].astype(np.int64), [int(s[2])]])


def _ur(users, items):
    ur = {}
    for u, i in zip(np.asarray(users).tolist(), np.asarray(items).tolist()):
        ur.setdefault(int(u), set()).add(int(i))
    return ur


def test_sampler_vs_fixture():
    from daisyrec_b200.utils.sampler import SkipGramNegativeSampler
    g = golden("item2vec")
    for k in range(int(g["n_synthetic"])):
        U, I, w, discard, seed = (int(v) for v in g[f"s{k}_meta"])
        users, items = g[f"s{k}_users"], g[f"s{k}_items"]
        ur = _ur(users, items)
        for u, i in g[f"s{k}_extra_ur"].tolist():
            ur.setdefault(u, set()).add(i)
        cfg = _config(user_num=U, item_num=I, train_ur=ur, context_window=w)
        np.random.seed(seed)
        rows = SkipGramNegativeSampler(_df(users, items), cfg, discard=bool(discard)).sampling()
        assert rows.dtype == np.int64 and np.array_equal(rows, g[f"s{k}_rows"].astype(np.int64)), k
        assert np.array_equal(_state(), g[f"s{k}_state"]), k
    # a user with contexts and no item left to draw: numpy's ValueError
    users, items = [0, 0, 1, 1], [0, 1, 0, 2]
    cfg = _config(user_num=2, item_num=2, train_ur={0: {0, 1}, 1: {0}})
    with pytest.raises(ValueError, match="cannot be empty"):
        SkipGramNegativeSampler(_df(users, items), cfg).sampling()


def test_sampler_vs_oracle_large():
    from daisyrec_b200.utils.sampler import SkipGramNegativeSampler
    rng = np.random.default_rng(3)
    U, I, n, w = 2000, 3000, 200_000, 3
    users = rng.integers(0, U, n)
    users[:20_000] = 17                                            # one user longer than the shared-memory sort
    items = np.minimum(rng.zipf(1.2, n) - 1, I - 1)
    ur = _ur(users, items)
    cfg = _config(user_num=U, item_num=I, train_ur=ur, context_window=w)
    np.random.seed(5)
    rows = SkipGramNegativeSampler(_df(users, items), cfg).sampling()
    st = _state()
    np.random.seed(5)
    want = io.skipgram_rows(io.group_sequences(users, items), ur, I, w)
    assert rows.shape == want.shape and np.array_equal(rows, want)
    assert np.array_equal(st, _state())


@pytest.mark.parametrize("opt", ["sgd", "adam"])
@pytest.mark.parametrize("B", [1, 255, 4096, 65573])
def test_step_vs_oracle(opt, B):
    from daisyrec_b200 import ops
    rng = np.random.default_rng(B)
    I, F, lr = 3000, 100, 0.05
    n = 3 * B - (B // 3)                                           # ragged last batch
    rows = np.stack([rng.integers(0, I, n), rng.integers(0, I, n), rng.integers(0, 2, n)], 1)
    rows[::7, 1] = rows[::7, 0]                                    # t == c
    Q0 = (rng.standard_normal((I, F)) * 0.1).astype(np.float32)
    Q = torch.from_numpy(Q0).cuda()
    ws = ops.I2VWorkspace(I, F, opt, Q.device)
    d = torch.from_numpy(rows.astype(np.int32)).cuda()
    bt, bc, bl = (d[:, k].contiguous() for k in range(3))
    losses = ops.i2v_train_steps(Q, ws, bt, bc, bl, B, 0, 3, ops.hyper(lr, 0., 0., opt, loss='CL')).cpu().numpy()
    Qo = Q0.astype(np.float64)
    adam = (np.zeros_like(Qo), np.zeros_like(Qo))
    want = [io.i2v_step(Qo, rows[s * B:(s + 1) * B], lr, opt, adam, s + 1) for s in range(3)]
    assert np.allclose(losses, want, rtol=2e-6, atol=1e-6)
    err = np.abs(Q.cpu().numpy() - Qo)
    if opt == "sgd":
        assert err.max() <= 1e-5
    else:
        moved = np.abs(adam[0]) > 1e-4 * np.abs(adam[0]).max()
        assert err[moved].max() <= 1e-4 and err.max() <= 3 * lr * 1.01


def _model(U=8, I=20, **kw):
    from daisyrec_b200.model.Item2VecRecommender import Item2Vec
    ur = {0: {1, 2, 3}, 1: {4, 5}, 2: {6}}
    torch.manual_seed(0)
    return Item2Vec(_config(user_num=U, item_num=I, train_ur=ur, **kw))


def test_calc_loss_errors():
    m = _model()
    Q0 = m.shared_embedding.weight.clone()
    batch = (torch.tensor([1, 2, 3]), torch.tensor([2, 2, 9]), torch.tensor([1, 0, 1]))
    loss = m.calc_loss(batch)
    x = (Q0[[1, 2, 3]] * Q0[[2, 2, 9]]).sum(1).double().cpu()
    y = torch.tensor([1., 0., 1.], dtype=torch.float64)
    want = torch.nn.functional.binary_cross_entropy_with_logits(x, y, reduction='sum')
    assert loss.shape == () and abs(float(loss) - float(want)) <= 1e-6 * abs(float(want)) + 1e-7
    assert torch.equal(m.shared_embedding.weight, Q0)              # no update
    with pytest.raises(IndexError):
        m.calc_loss((torch.tensor([1]), torch.tensor([20]), torch.tensor([1])))
    m.shared_embedding.weight[2, 0] = float('nan')
    with pytest.raises(ValueError):
        m.calc_loss(batch)


def test_fit_keeps_rows_of_users_without_train_rows():
    from daisyrec_b200.utils.dataset import BasicDataset, get_dataloader
    m = _model()
    P0 = m.user_embedding.weight.clone()
    rows = np.array([[1, 2, 1], [2, 1, 1], [1, 7, 0], [2, 11, 0], [4, 5, 1], [5, 4, 1], [4, 0, 0], [5, 19, 0]], np.int64)
    m.fit(get_dataloader(BasicDataset(rows), batch_size=3, shuffle=True, num_workers=0))
    P, Q = m.user_embedding.weight.cpu(), m.shared_embedding.weight.cpu()
    assert torch.equal(P[3:], P0[3:].cpu())
    for u, items in {0: [1, 2, 3], 1: [4, 5], 2: [6]}.items():
        assert torch.allclose(P[u], Q[items].sum(0), rtol=1e-6, atol=1e-7)
    with pytest.raises(IndexError):                                # column 0 is an item id here
        m.fit(get_dataloader(BasicDataset(np.array([[20, 1, 1]], np.int64)), batch_size=1, shuffle=False, num_workers=0))


def test_ml100k_driver_sequence():
    """test.py's item2vec branch through the drop-in classes: construct -> sample -> fit -> rank on the reference's
    candidate sets."""
    from daisyrec_b200.model.Item2VecRecommender import Item2Vec
    from daisyrec_b200.utils.sampler import SkipGramNegativeSampler
    from daisyrec_b200.utils.dataset import BasicDataset, CandidatesDataset, get_dataloader
    from daisyrec_b200.utils.utils import get_ur, build_candidates_set
    g, gs, gr = golden("item2vec"), golden("ml100k_sampler"), golden("ml100k_rank")
    U, I, F, w, seed, B, T, stride = (int(v) for v in g["ml_meta"])
    train_set = _df(gs["coo_u"], gs["coo_i"])                     # config 1's split, as the fixture's run
    off = np.concatenate([[0], np.cumsum(gr["gt_len"])])
    test_ur = {int(u): gr["gt_flat"][off[k]:off[k + 1]].tolist() for k, u in enumerate(gr["test_u"])}
    cfg = _config(user_num=U, item_num=I, factors=F, context_window=w, batch_size=B, lr=float(g["ml_lr"]))
    np.random.seed(seed); torch.manual_seed(seed)
    train_ur = get_ur(train_set)
    cfg['train_ur'] = train_ur
    model = Item2Vec(cfg)
    P0 = model.user_embedding.weight.cpu().numpy().copy()
    assert hashlib.sha256(P0.tobytes()).digest() == g["ml_P0_sha"].tobytes()
    assert hashlib.sha256(model.shared_embedding.weight.cpu().numpy().tobytes()).digest() == g["ml_Q0_sha"].tobytes()
    rows = SkipGramNegativeSampler(train_set, cfg).sampling()
    assert rows.dtype == np.int64 and rows.shape == (T, 3)
    assert hashlib.sha256(np.ascontiguousarray(rows).tobytes()).digest() == g["ml_rows_sha"].tobytes()
    assert np.array_equal(_state(), g["ml_state"])
    losses = []
    orig = model._train_steps

    def rec(*a):
        out = orig(*a)
        losses.append(out.cpu().numpy())
        return out

    model._train_steps = rec
    model.fit(get_dataloader(BasicDataset(rows), batch_size=B, shuffle=True, num_workers=4))
    losses = np.concatenate(losses)
    want = g["ml_fit_losses"]
    print(f"epoch loss {losses.sum():.6f} vs {want.sum():.6f}; worst step rel "
          f"{np.max(np.abs(losses - want) / np.abs(want)):.2e}")
    assert losses.shape == want.shape and abs(losses.sum() - want.sum()) <= 1e-5 * abs(want.sum())
    Q, P = model.shared_embedding.weight.cpu().numpy(), model.user_embedding.weight.cpu().numpy()
    eq, ep = np.abs(Q - g["ml_fit_Q"]), np.abs(P[::stride] - g["ml_fit_P"])
    print(f"shared max {eq.max():.2e} p99.9 {np.quantile(eq, 0.999):.2e}; user max {ep.max():.2e} rel "
          f"{ep.max() / np.abs(g['ml_fit_P']).max():.2e}")
    assert eq.max() < 1e-3 and np.quantile(eq, 0.999) < 1e-4
    assert ep.max() < 1e-3 * max(1.0, np.abs(g["ml_fit_P"]).max())
    missing = [u for u in range(U) if u not in train_ur]
    assert np.array_equal(P[missing], P0[missing])
    test_u, test_ucands = build_candidates_set(test_ur, train_ur, cfg)   # test.py:112
    cands = np.stack([c[1] for c in test_ucands])
    assert hashlib.sha256(cands.tobytes()).digest() == g["ml_cands_sha"].tobytes()
    preds = model.rank(get_dataloader(CandidatesDataset(test_ucands), batch_size=128, shuffle=False, num_workers=0))
    assert preds.dtype == np.float32 and preds.shape == g["ml_preds"].shape
    same = (preds == g["ml_preds"]).mean()
    print(f"rank position-equal {same:.4f}")
    assert same >= 0.97
    full = np.stack([model.full_rank(int(u)) for u in test_u[:4]])
    assert full.dtype == np.int64 and (full == g["ml_full"]).mean() >= 0.9
    assert abs(model.predict(test_u[0], int(cands[0][-1])) - float(g["ml_predict"][0])) <= 1e-3 * abs(float(g["ml_predict"][0])) + 1e-4
