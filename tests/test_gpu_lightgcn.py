"""GPU parity for LightGCN (SURVEY 8(a) row a15): golden fixtures from the reference + oracle on random graphs."""
import logging

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from conftest import golden

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from daisyrec_b200 import ops as o
    o.require_cuda()
    return o


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def test_lightgcn_golden(ops, orc):
    g = golden("lightgcn")
    for c in range(int(g["ncases"])):
        U, I, F, L, lr, r1, r2, opt = g[f"c{c}_hyper"]
        U, I, F, L = int(U), int(I), int(F), int(L)
        optn = "sgd" if opt == 0 else "adam"
        row_ptr, col, val = ops.lgcn_norm_adj(g[f"c{c}_coo_u"], g[f"c{c}_coo_i"], U, I)
        assert np.array_equal(val, g[f"c{c}_adj_val"]) and np.array_equal(col, g[f"c{c}_adj_idx"][1])
        graph = ops.LgcnGraph(row_ptr, col, val, "cuda")
        E, bs, losses = g[f"c{c}_E"], g[f"c{c}_batches"], g[f"c{c}_loss"]
        ws = ops.LgcnWorkspace(U, I, F, optn, "cuda")
        E0 = dev(E[0])
        Em0 = ops.lgcn_propagate(E0, ws, graph, L).cpu().numpy()
        np.testing.assert_allclose(Em0, g[f"c{c}_Em0"], rtol=0, atol=3e-7 * max(1.0, np.abs(Em0).max()))
        hp = ops.hyper(lr, r1, r2, optn)
        # chained: 3 steps from the reference's initial state (Adam moments evolve inside the workspace)
        for s in range(bs.shape[0]):
            b = [dev(bs[s][k]) for k in range(3)]
            l0 = ops.lgcn_bpr_train_steps(E0, ws, graph, L, *b, b[0].numel(), 0, 1, hp, apply=False).item()
            loss = ops.lgcn_bpr_train_steps(E0, ws, graph, L, *b, b[0].numel(), 0, 1, hp, adam_step0=s).item()
            assert abs(l0 - losses[s]) <= 2e-5 * abs(losses[s]) and abs(loss - losses[s]) <= 2e-5 * abs(losses[s])
            tol = (5e-6 if opt == 0 else 1e-4) * (s + 1)
            np.testing.assert_allclose(E0.cpu().numpy(), E[s + 1], rtol=0, atol=tol * max(1.0, np.abs(E[s + 1]).max()))
        # ranking on the reference's propagated tables: bit-exact ids
        Emf = g[f"c{c}_Em_final"]
        users, cands = g[f"c{c}_users"], g[f"c{c}_cands"].astype(np.int64)
        got = ops.mf_rank(dev(Emf[:U]), dev(Emf[U:]), dev(users), dev(cands), 10).cpu().numpy()
        assert np.array_equal(got, g[f"c{c}_preds"])


@pytest.mark.parametrize("F,L,opt,reg", [(64, 3, "adam", 0.0), (32, 2, "sgd", 0.001), (100, 2, "adam", 0.002), (8, 1, "sgd", 0.0)])
def test_lightgcn_vs_oracle_random(ops, orc, F, L, opt, reg):
    rng = np.random.default_rng(F * 10 + L)
    U, I, nnz, B = 700, 500, 12000, 2048
    cu = rng.integers(U, size=nnz).astype(np.int32)
    ci = np.minimum(I - 1, rng.zipf(1.15, size=nnz) - 1).astype(np.int32)   # a few items with >256 neighbours
    row_ptr, col, val = ops.lgcn_norm_adj(cu, ci, U, I)
    assert np.diff(row_ptr).max() > 256                              # multi-segment rows are exercised
    rp2, col2, val2 = orc.lgcn_norm_adj(cu, ci, U, I)
    assert np.array_equal(row_ptr, rp2) and np.array_equal(col, col2) and np.array_equal(val, val2)
    graph = ops.LgcnGraph(row_ptr, col, val, "cuda")
    E0h = (rng.standard_normal((U + I, F)) * 0.2).astype(np.float32)
    Eo = E0h.copy()
    E0 = dev(E0h)
    ws = ops.LgcnWorkspace(U, I, F, opt, "cuda")
    hp_d, hp_o = ops.hyper(0.01, reg, reg, opt), orc.hyper(0.01, reg, reg, opt)
    Em = ops.lgcn_propagate(E0, ws, graph, L).cpu().numpy()
    np.testing.assert_allclose(Em, orc.lgcn_propagate(row_ptr, col, val, E0h, L), rtol=0, atol=2e-6)
    adam = None if opt == "sgd" else (np.zeros_like(Eo), np.zeros_like(Eo))
    for s in range(3):
        b = [rng.integers(U, size=B).astype(np.int32), rng.integers(I, size=B).astype(np.int32),
             rng.integers(I, size=B).astype(np.int32)]
        lo = orc.lgcn_bpr_step(Eo, U, I, L, row_ptr, col, val, *b, hp_o, True, adam, s + 1)
        ld = ops.lgcn_bpr_train_steps(E0, ws, graph, L, *[dev(x) for x in b], B, 0, 1, hp_d, adam_step0=s).item()
        assert abs(ld - lo) <= 5e-6 * abs(lo)
        np.testing.assert_allclose(E0.cpu().numpy(), Eo, rtol=0, atol=(1e-5 if opt == "sgd" else 2e-4))


def test_lightgcn_dropin_class(ops, orc):
    """The reference's call sequence (test.py:88-95,118-120) on the GPU-path LightGCN class."""
    from daisyrec_b200.model.LightGCNRecommender import LightGCN
    from daisyrec_b200.utils.dataset import BasicDataset, CandidatesDataset, get_dataloader
    g = golden("lightgcn")
    c = 1
    U, I, F, L, lr, r1, r2, opt = g[f"c{c}_hyper"]
    U, I, F, L = int(U), int(I), int(F), int(L)
    cu, ci = g[f"c{c}_coo_u"], g[f"c{c}_coo_i"]
    inter = sp.coo_matrix((np.ones(len(cu)), (cu, ci)), shape=(U, I))
    cfg = dict(gpu='', logger=logging.getLogger('t'), epochs=1, lr=lr, topk=10, user_num=U, item_num=I, inter_matrix=inter,
               factors=F, num_layers=L, reg_1=r1, reg_2=r2, loss_type='BPR', optimizer='default', init_method='default',
               early_stop=False, progress=False)
    torch.manual_seed(22)
    model = LightGCN(cfg)
    assert np.array_equal(model.E0.cpu().numpy(), g[f"c{c}_E"][0])          # same init stream as the reference
    bs = g[f"c{c}_batches"]
    data = np.ascontiguousarray(np.concatenate([bs[s].T for s in range(3)]))
    model.fit(get_dataloader(BasicDataset(data), batch_size=bs.shape[2], shuffle=False))
    np.testing.assert_allclose(model.E0.cpu().numpy(), g[f"c{c}_E"][3], rtol=0, atol=3e-4)
    users, cands = g[f"c{c}_users"], g[f"c{c}_cands"].astype(np.int64)
    loader = get_dataloader(CandidatesDataset([[int(u), cc] for u, cc in zip(users, cands)]), batch_size=128, shuffle=False)
    preds = model.rank(loader)
    assert preds.dtype == np.float32 and preds.shape == (9, 10)
    model.load_state_dict({'embed_user.weight': dev(g[f"c{c}_E"][3][:U]), 'embed_item.weight': dev(g[f"c{c}_E"][3][U:])})
    assert (model.rank(loader) == g[f"c{c}_preds"]).mean() > 0.97            # propagated tables differ by fp32 noise
    assert model.full_rank(int(users[0])).dtype == np.int64
    assert abs(model.predict(int(users[0]), int(cands[0][0])) - float(g[f"c{c}_pred_pair"][0])) < 1e-5
