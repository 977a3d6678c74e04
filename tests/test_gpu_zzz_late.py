"""Tests of CUDA paths written after the round's last GPU slot (this file sorts last on purpose):
* NFM with nn.Dropout active (the reference default, assets/nfm.yaml: dropout 0.5) and NGCF with its message dropout (default
  0.1) against reference-generated fixtures (tests/golden/nfm_dropout.npz, ngcf_dropout.npz): the host draws torch's own masks in
  the reference's order, the kernels apply them;
* the KPI impact of the fused bf16 NeuMF tower on a config-1-sized run."""
import logging

import numpy as np
import pytest
import torch

from conftest import golden

pytestmark = pytest.mark.gpu
ACTS = ["relu", "sigmoid", "tanh"]


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _keep_bytes(B, F, L, p):
    """torch's draws for one step, in the reference's order -> (uint8 CUDA tensor for the kernels, float factors for the oracle)."""
    parts = []
    for _side in (0, 1):
        for _site in range(1 + L):
            parts.append(torch.empty(B, F, dtype=torch.float32).bernoulli_(1.0 - p))
    k = torch.stack(parts).reshape(2, 1 + L, B, F)
    scale = np.float32(1.0) / np.float32(1.0 - p)
    f = k.numpy() * scale
    return k.to(torch.uint8).reshape(-1).cuda(), (np.ascontiguousarray(f[0], np.float32), np.ascontiguousarray(f[1], np.float32))


def test_nfm_dropout_steps_match_reference_fixture(orc):
    from daisyrec_b200 import ops
    g = golden("nfm_dropout")
    for c in range(int(g["ncases"])):
        L, bn, act, lr, r1, r2, opt, drop, seed = g[f"c{c}_hyper"]
        L, bn, act, seed, drop = int(L), bool(bn), int(act), int(seed), float(drop)
        optn = "sgd" if opt == 0 else "adam"
        Ps, Qs, Bs, Ns, Rs = g[f"c{c}_P"], g[f"c{c}_Q"], g[f"c{c}_bias"], g[f"c{c}_N"], g[f"c{c}_R"]
        bs, losses = g[f"c{c}_batches"], g[f"c{c}_loss"]
        U, F = Ps.shape[1:]
        I = Qs.shape[1]
        hp = ops.hyper(float(lr), float(r1), float(r2), optn)
        ho = orc.hyper(lr=lr, reg_1=r1, reg_2=r2, opt=optn)
        ws = ops.NfmWorkspace(U, I, F, L, bn, optn, 2 * bs.shape[2], "cuda")       # optimiser state carried across the steps
        tot = Ps[0].size + Qs[0].size + Bs.shape[1] + Ns.shape[1]
        state = None if opt == 0 else np.zeros(2 * tot, np.float32)
        torch.manual_seed(seed + 100)
        for s in range(bs.shape[0]):
            P, Q, bias, N = dev(Ps[s]), dev(Qs[s]), dev(Bs[s]), dev(Ns[s])
            R = dev(Rs[s]) if bn else None
            b = [dev(bs[s][k]) for k in range(3)]
            keep_d, keep_h = _keep_bytes(b[0].numel(), F, L, drop)
            loss = ops.nfm_bpr_train_steps(P, Q, bias, N, R, ws, act, *b, b[0].numel(), 0, 1, hp, adam_step0=s, dropout=drop,
                                           keep=keep_d).item()
            assert abs(loss - losses[s]) <= 3e-5 * abs(losses[s]), (c, s, loss, losses[s])
            # the oracle on the same masks (pinned on this fixture by tests/test_oracle_golden.py)
            Po, Qo, bo, No, Ro = (a[s].copy() for a in (Ps, Qs, Bs, Ns, Rs))
            bh = np.ascontiguousarray(bs[s])
            lo = orc.nfm_bpr_step(Po, Qo, bo, No, Ro, L, bn, act, bh[0], bh[1], bh[2], ho, True, state, s + 1, keep=keep_h)
            assert abs(loss - lo) <= 3e-5 * abs(lo), (c, s, loss, lo)
            for got, want, nm in ((P, Ps[s + 1], "P"), (Q, Qs[s + 1], "Q"), (bias, Bs[s + 1], "bias"), (N, Ns[s + 1], "N")):
                err = np.abs(got.cpu().numpy() - want)
                tol = (1e-5 if optn == "sgd" else 1e-4) * max(1.0, np.abs(want).max())
                assert (err <= tol).mean() >= 0.99 and err.max() <= 2.1 * float(lr) + tol, \
                    (c, s, nm, float((err <= tol).mean()), float(err.max()))
            if bn:
                np.testing.assert_allclose(R.cpu().numpy(), Rs[s + 1], rtol=2e-5, atol=2e-6, err_msg=f"running stats {c} {s}")
        assert np.array_equal(torch.get_rng_state().numpy(), g[f"c{c}_rng_after"]), c   # as many draws as the reference made


def test_nfm_class_runs_the_reference_default_config():
    """NFM(config) with the reference's default dropout: three train_step calls from the fixture's state reproduce the
    reference's parameters and leave torch's global generator where the reference left it; eval-mode ranking has no dropout."""
    from daisyrec_b200.model import NFM
    from daisyrec_b200.utils.dataset import CandidatesDataset, get_dataloader
    g = golden("nfm_dropout")
    for c in range(int(g["ncases"])):
        L, bn, act, lr, r1, r2, opt, drop, seed = g[f"c{c}_hyper"]
        L, bn, act, seed = int(L), bool(bn), int(act), int(seed)
        U, F = g[f"c{c}_P"].shape[1:]
        I = g[f"c{c}_Q"].shape[1]
        cfg = dict(gpu="", logger=logging.getLogger("t"), epochs=1, lr=float(lr), reg_1=float(r1), reg_2=float(r2), user_num=U,
                   item_num=I, factors=F, num_layers=L, batch_norm=bn, act_function=ACTS[act], dropout=float(drop), loss_type="BPR",
                   optimizer="sgd" if opt == 0 else "adam", init_method="default", early_stop=False, topk=10, progress=False)
        torch.manual_seed(seed)
        m = NFM(cfg)
        Bs = g[f"c{c}_bias"]
        sd = {"embed_user.weight": g[f"c{c}_P"][0], "embed_item.weight": g[f"c{c}_Q"][0], "u_bias.weight": Bs[0][:U],
              "i_bias.weight": Bs[0][U:U + I], "bias_": Bs[0][U + I:], "net": g[f"c{c}_N"][0]}
        if bn:
            sd["running"] = g[f"c{c}_R"][0]
        m.load_state_dict(sd)
        b = g[f"c{c}_batches"]
        torch.manual_seed(seed + 100)
        for s in range(3):
            loss = m.train_step([torch.from_numpy(b[s][k]) for k in range(3)])
            assert abs(loss - g[f"c{c}_loss"][s]) <= (5e-5 if opt == 0 else 2e-3) * abs(g[f"c{c}_loss"][s]), (c, s, loss)
        assert np.array_equal(torch.get_rng_state().numpy(), g[f"c{c}_rng_after"]), c
        want = g[f"c{c}_P"][3]
        err = np.abs(m.embed_user.weight.cpu().numpy() - want)
        tol = (3e-5 if opt == 0 else 3e-4) * max(1.0, np.abs(want).max())
        assert (err <= tol).mean() >= 0.98, (c, float((err <= tol).mean()))
        # eval mode: no dropout, running statistics -- the reference's ranking on its own final state
        m.load_state_dict({"embed_user.weight": g[f"c{c}_P"][3], "embed_item.weight": g[f"c{c}_Q"][3], "u_bias.weight": Bs[3][:U],
                           "i_bias.weight": Bs[3][U:U + I], "bias_": Bs[3][U + I:], "net": g[f"c{c}_N"][3],
                           **({"running": g[f"c{c}_R"][3]} if bn else {})})
        m.eval()
        users, cands = g[f"c{c}_users"], g[f"c{c}_cands"].astype(np.int64)
        loader = get_dataloader(CandidatesDataset([[int(u), cands[r]] for r, u in enumerate(users)]), batch_size=128, shuffle=False)
        preds = m.rank(loader)
        assert (preds == g[f"c{c}_preds"]).mean() >= 0.97, c
        with pytest.raises(ValueError):
            NFM(dict(cfg, dropout=1.0))


# ------------------------------------------------------------------ NGCF message dropout (reference default mess_dropout 0.1)
def _ngcf_keep(n, dims, p):
    parts = [torch.empty(n, int(d), dtype=torch.float32).bernoulli_(1.0 - p) for d in list(dims)[1:]]
    flat = torch.cat([t.reshape(-1) for t in parts])
    scale = np.float32(1.0) / np.float32(1.0 - p)
    return flat.to(torch.uint8).cuda(), np.ascontiguousarray(flat.numpy() * scale, np.float32)


def test_ngcf_message_dropout_matches_reference_fixture(orc):
    from daisyrec_b200 import ops
    g = golden("ngcf_dropout")
    for c in range(int(g["ncases"])):
        U, I, lr, r1, r2, opt, drop, seed = g[f"c{c}_hyper"]
        U, I, seed, drop = int(U), int(I), int(seed), float(drop)
        optn = "sgd" if opt == 0 else "adam"
        dims = [int(d) for d in g[f"c{c}_dims"]]
        row_ptr, col, val = ops.lgcn_norm_adj(g[f"c{c}_coo_u"], g[f"c{c}_coo_i"], U, I)
        graph = ops.LgcnGraph(row_ptr, col, val, "cuda")
        Es, Ws, bs, losses = g[f"c{c}_E"], g[f"c{c}_W"], g[f"c{c}_batches"], g[f"c{c}_loss"]
        ws = ops.NgcfWorkspace(U, I, dims, optn, "cuda")
        torch.manual_seed(seed + 50)
        keep_d, _ = _ngcf_keep(U + I, dims, drop)
        rep = ops.ngcf_forward(dev(Es[0]), dev(Ws[0]), ws, graph, dropout=drop, keep=keep_d).cpu().numpy()
        np.testing.assert_allclose(rep, g[f"c{c}_all0"], rtol=0, atol=3e-6, err_msg=f"case {c} forward")
        hp = ops.hyper(lr, r1, r2, optn)
        ho = orc.hyper(lr=lr, reg_1=r1, reg_2=r2, opt=optn)
        state = None if opt == 0 else np.zeros(2 * (Es[0].size + Ws.shape[1]), np.float32)
        torch.manual_seed(seed + 100)
        for s in range(bs.shape[0]):
            E, W = dev(Es[s]), dev(Ws[s])
            b = [dev(bs[s][k]) for k in range(3)]
            keep_d, keep_h = _ngcf_keep(U + I, dims, drop)
            l1 = ops.ngcf_bpr_train_steps(E, W, ws, graph, *b, b[0].numel(), 0, 1, hp, adam_step0=s, dropout=drop, keep=keep_d).item()
            assert abs(l1 - losses[s]) <= 3e-5 * abs(losses[s]), (c, s, l1, losses[s])
            Eo, Wo = Es[s].copy(), Ws[s].copy()
            bh = np.ascontiguousarray(bs[s])
            lo = orc.ngcf_bpr_step(Eo, Wo, U, I, np.asarray(dims, np.int32), row_ptr, col, val, bh[0], bh[1], bh[2], ho, True, state,
                                   s + 1, keep=keep_h)
            assert abs(l1 - lo) <= 3e-5 * abs(lo), (c, s, l1, lo)
            for got, want, nm in ((E.cpu().numpy(), Es[s + 1], "E"), (W.cpu().numpy(), Ws[s + 1], "W")):
                err = np.abs(got - want)
                tol = (5e-6 if optn == "sgd" else 5e-5) * max(1.0, np.abs(want).max())
                assert (err <= tol).mean() >= 0.99 and err.max() <= 2.1 * lr + tol, (c, s, nm, float((err <= tol).mean()), float(err.max()))
        assert np.array_equal(torch.get_rng_state().numpy(), g[f"c{c}_rng_after"]), c


def test_ngcf_class_runs_the_reference_default_config():
    """NGCF(config) with the reference's default mess_dropout: train steps from the fixture's state, then rank() -- whose
    forward() still drops, as the reference's does -- reproduce the reference from the same generator seeds."""
    import pandas as pd
    from daisyrec_b200.model import NGCF
    from daisyrec_b200.utils.dataset import CandidatesDataset, get_dataloader
    from daisyrec_b200.utils.utils import get_inter_matrix
    g = golden("ngcf_dropout")
    for c in range(int(g["ncases"])):
        U, I, lr, r1, r2, opt, drop, seed = g[f"c{c}_hyper"]
        U, I, seed = int(U), int(I), int(seed)
        dims = [int(d) for d in g[f"c{c}_dims"]]
        cu, ci = g[f"c{c}_coo_u"], g[f"c{c}_coo_i"]
        df = pd.DataFrame({"user": cu, "item": ci, "rating": 1.0, "timestamp": np.arange(len(cu))})
        cfg = dict(gpu="", logger=logging.getLogger("t"), epochs=1, lr=float(lr), reg_1=float(r1), reg_2=float(r2), user_num=U,
                   item_num=I, factors=dims[0], hidden_size_list=dims[1:], node_dropout=0.0, mess_dropout=float(drop),
                   loss_type="BPR", optimizer="sgd" if opt == 0 else "default", init_method="default", early_stop=False, topk=10,
                   progress=False, UID_NAME="user", IID_NAME="item", INTER_NAME="rating")
        cfg["inter_matrix"] = get_inter_matrix(df, cfg)
        torch.manual_seed(seed)
        m = NGCF(cfg)
        assert np.array_equal(m.E0.cpu().numpy(), g[f"c{c}_E"][0]) and np.array_equal(m.gnn.cpu().numpy(), g[f"c{c}_W"][0]), c
        torch.manual_seed(seed + 50)
        eu, ei = m.forward()
        np.testing.assert_allclose(torch.cat([eu, ei]).cpu().numpy(), g[f"c{c}_all0"], rtol=0, atol=3e-6)
        b = g[f"c{c}_batches"]
        torch.manual_seed(seed + 100)
        for s in range(3):
            loss = m.train_step([torch.from_numpy(b[s][k]) for k in range(3)])
            assert abs(loss - g[f"c{c}_loss"][s]) <= (5e-5 if opt == 0 else 3e-3) * abs(g[f"c{c}_loss"][s]), (c, s, loss)
        assert np.array_equal(torch.get_rng_state().numpy(), g[f"c{c}_rng_after"]), c
        m.load_state_dict({"embed_user.weight": g[f"c{c}_E"][3][:U], "embed_item.weight": g[f"c{c}_E"][3][U:], "gnn": g[f"c{c}_W"][3]})
        users, cands = g[f"c{c}_users"], g[f"c{c}_cands"].astype(np.int64)
        loader = get_dataloader(CandidatesDataset([[int(u), cands[r]] for r, u in enumerate(users)]), batch_size=128, shuffle=False)
        torch.manual_seed(seed + 200)
        preds = m.rank(loader)
        np.testing.assert_allclose(torch.cat([m.restore_user_e, m.restore_item_e]).cpu().numpy(), g[f"c{c}_all_rank"], rtol=0, atol=3e-6)
        assert (preds == g[f"c{c}_preds"]).mean() >= 0.97, c


# ------------------------------------------------------------------ KPI impact of the bf16 / fused NeuMF tower (config-1-sized run)
def test_neumf_fused_tower_kpi_impact_is_small():
    """NeuMF (F = 32, tower 128 -> 64 -> 32, Adam, dropout 0) trained for two epochs on the ML-100K fixture triples (the config-1
    data: 943 x 1 152, 313 452 triples, batch 256) from the same initial weights and the same batch order, once with the fp32
    tower and once with the fused bf16 wgmma tower: NDCG@10 / HR@10 on the fixture's 304 test users x 1 000 candidates move by
    less than the stated bound (bf16 rounds every product operand to 8 bits of mantissa; the gap is training noise, not bias)."""
    from daisyrec_b200 import ops
    from daisyrec_b200.model import NeuMF
    from daisyrec_b200.utils.dataset import BasicDataset, CandidatesDataset, get_dataloader
    gs, gr = golden("ml100k_sampler"), golden("ml100k_rank")
    U, I, G, _seed = (int(v) for v in gs["meta"])
    samples = np.stack([np.repeat(gs["coo_u"].astype(np.int32), G), np.repeat(gs["coo_i"].astype(np.int32), G),
                        gs["triples_j"].astype(np.int32)], 1)
    users, cands = gr["test_u"].astype(np.int64), gr["cands"].astype(np.int64)
    test_loader = get_dataloader(CandidatesDataset([[int(u), cands[r]] for r, u in enumerate(users)]), batch_size=128, shuffle=False)
    gt_ptr = torch.from_numpy(np.concatenate([[0], np.cumsum(gr["gt_len"])]).astype(np.int64)).cuda()
    off = np.concatenate([[0], np.cumsum(gr["gt_len"])])
    gt_idx = torch.from_numpy(np.concatenate([np.sort(gr["gt_flat"][off[k]:off[k + 1]]) for k in range(len(users))]).astype(np.int32)).cuda()
    kpi = {}
    for tower in ("fp32", "fused"):
        cfg = dict(gpu='', logger=logging.getLogger('t'), lr=0.001, epochs=2, reg_1=0.0, reg_2=0.0, dropout=0.0, model_name='NeuMF',
                   GMF_model=None, MLP_model=None, user_num=U, item_num=I, factors=32, num_layers=2, loss_type='BPR',
                   optimizer='default', init_method='default', early_stop=False, topk=10, progress=False, tower_dtype=tower)
        torch.manual_seed(2022)
        m = NeuMF(cfg)
        m.fit(get_dataloader(BasicDataset(samples), batch_size=256, shuffle=True))
        preds = torch.from_numpy(np.ascontiguousarray(m.rank(test_loader), np.float32)).cuda()
        res = ops.rank_metrics(preds, gt_ptr, gt_idx, [10], I).cpu().numpy()[0]
        kpi[tower] = {"ndcg": float(res[2]), "hr": float(res[3])}
    print("NeuMF KPI impact (NDCG@10, HR@10):", kpi)
    assert kpi["fp32"]["ndcg"] > 0.02 and kpi["fused"]["ndcg"] > 0.02, kpi        # both models learned something
    assert abs(kpi["fp32"]["ndcg"] - kpi["fused"]["ndcg"]) <= 0.03 and abs(kpi["fp32"]["hr"] - kpi["fused"]["hr"]) <= 0.06, kpi


# ------------------------------------------------------------------ MT19937 from many CTAs (jump-ahead), every table level
def test_mt19937_stream_across_all_jump_levels():
    """drb_mt19937_stream == numpy's MT19937 for a stream long enough to need every level of csrc/mt_jump_table.inc (129 segments
    of 1 680 blocks: segment 128 takes level 7, segment 127 takes levels 0-6), whichever kernel the one-off device check selected."""
    from daisyrec_b200 import ops
    seg = 1680 * 624
    n = 128 * seg + 5 * 624 + 77
    print("mt19937 kernel for", n, "words:", ops.mt19937_stream_variant(n))
    got = ops.mt19937_stream(424242, n, "cuda")
    rs = np.random.RandomState(424242)
    for lo in range(0, n, 1 << 24):
        hi = min(n, lo + (1 << 24))
        want = np.frombuffer(rs.bytes(4 * (hi - lo)), dtype="<u4")
        assert np.array_equal(got[lo:hi].cpu().numpy().view(np.uint32), want), (lo, hi)
    # and a short stream stays on the one-CTA kernel
    assert ops.mt19937_stream_variant(1000) == "one-cta"
