"""GPU parity tests (run with -m gpu on an H100): the CUDA path, called through the C ABI
(daisyrec_b200.ops -> libdaisyrec_b200.so), against the golden fixtures of the real reference and
against the CPU oracle on seeded random inputs.

Bars: bit-exact for integer/index work (js tables, triples, candidate top-K ids); fp32 work within
the tolerances written below (north_star: loss within 1e-4).
"""
import numpy as np
import pytest
import torch

from conftest import golden, csr_from_coo

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from daisyrec_b200 import ops as o
    o.require_cuda()
    return o


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


# ------------------------------------------------------------------ sampler
def _sample_device(ops, seed_state, cu, ci, U, I, G):
    row_ptr, col = csr_from_coo(cu, ci, U)
    draws = ops.sampler_draw_mt19937(seed_state, row_ptr, U, I, G)
    js = ops.sampler_kth_complement(dev(row_ptr), dev(col), dev(draws), I)
    tr = ops.sampler_explode(dev(cu), dev(ci), js)
    return js.cpu().numpy(), tr.cpu().numpy()


def test_sampler_golden_small(ops):
    g = golden("sampler_small")
    for c in range(int(g["ncases"])):
        U, I, G, seed = (int(v) for v in g[f"c{c}_meta"])
        st = ops.mt19937_seed(seed)
        js, tr = _sample_device(ops, st, g[f"c{c}_coo_u"], g[f"c{c}_coo_i"], U, I, G)
        assert tr.dtype == np.int32 and np.array_equal(tr, g[f"c{c}_triples"])
        ops.mt19937_to_numpy(st)                                  # stream position == the reference's
        assert np.array_equal(np.random.randint(0, 2 ** 31 - 1, size=3), g[f"c{c}_next"])


def test_sampler_golden_ml100k_and_host_call(ops):
    g = golden("ml100k_sampler")
    U, I, G, seed = (int(v) for v in g["meta"])
    cu, ci = g["coo_u"].astype(np.int32), g["coo_i"].astype(np.int32)
    js, tr = _sample_device(ops, ops.mt19937_seed(seed), cu, ci, U, I, G)
    assert np.array_equal(tr[:, 2], g["triples_j"].astype(np.int32))
    assert np.array_equal(tr[:3], [[258, 246, 781], [258, 246, 640], [258, 246, 1050]])
    row_ptr, col = csr_from_coo(cu, ci, U)
    js2, tr2 = ops.sample_triples_host(ops.mt19937_seed(seed), row_ptr, col, cu, ci, U, I, G)
    assert np.array_equal(js2, js) and np.array_equal(tr2, tr)


def test_sampler_vs_oracle_random(ops, orc):
    rng = np.random.default_rng(3)
    U, I, G, nnz = 3000, 5000, 4, 200_000
    cu = rng.integers(U, size=nnz).astype(np.int32)
    ci = np.minimum(I - 1, rng.zipf(1.2, size=nnz) - 1).astype(np.int32)
    row_ptr, col = csr_from_coo(cu, ci, U)
    want_js = orc.sample_negatives(orc.mt_seed(77), row_ptr, col, U, I, G)
    js, tr = _sample_device(ops, ops.mt19937_seed(77), cu, ci, U, I, G)
    assert np.array_equal(js, want_js)
    assert np.array_equal(tr, orc.explode_triples(cu, ci, want_js))
    # property: no sampled negative is a positive of its user
    pos = set(zip(cu.tolist(), ci.tolist()))
    assert not any((int(u), int(j)) in pos for u, j in zip(tr[::97, 0], tr[::97, 2]))


def test_sampler_philox_properties(ops):
    rng = np.random.default_rng(4)
    U, I, G, nnz = 2000, 300, 8, 60_000
    cu = rng.integers(U, size=nnz).astype(np.int32)
    ci = rng.integers(I, size=nnz).astype(np.int32)
    row_ptr, col = csr_from_coo(cu, ci, U)
    draws, bad = ops.sampler_draw_philox(1234, 0, dev(row_ptr), U, I, G)
    js = ops.sampler_kth_complement(dev(row_ptr), dev(col), draws, I).cpu().numpy()
    assert int(bad.item()) > U                                   # no user without a complement
    deg = np.diff(row_ptr)
    d = draws.cpu().numpy()
    assert (d >= 0).all() and (d < (I - deg)[:, None]).all()
    pos = set(zip(cu.tolist(), ci.tolist()))
    assert not any((u, int(j)) in pos for u in range(0, U, 7) for j in js[u])
    assert (js >= 0).all() and (js < I).all()
    # uniformity smoke: mean of draws/(n) ~ 0.5
    assert abs((d / (I - deg)[:, None]).mean() - 0.5) < 0.02


def test_sampler_empty_complement(ops):
    row_ptr = np.array([0, 3], np.int64)
    with pytest.raises(ValueError):
        ops.sampler_draw_mt19937(ops.mt19937_seed(1), row_ptr, 1, 3, 2)


# ------------------------------------------------------------------ BPR step
def test_mf_steps_golden(ops):
    g = golden("mf_steps")
    for c in range(int(g["ncases"])):
        lr, r1, r2, opt, lk = g[f"c{c}_hyper"]
        optn = "sgd" if opt == 0 else "adam"
        Ps, Qs, bs, losses = g[f"c{c}_P"], g[f"c{c}_Q"], g[f"c{c}_batches"], g[f"c{c}_loss"]
        U, F = Ps[0].shape
        I = Qs[0].shape[0]
        hp = ops.hyper(lr, r1, r2, optn, loss=("BPR", "HL", "TL")[int(lk)])
        P, Q = dev(Ps[0]), dev(Qs[0])
        ws = ops.MFWorkspace(U, I, F, optn, "cuda")
        for s in range(bs.shape[0]):
            b = bs[s]
            bu, bi, bj = dev(b[0]), dev(b[1]), dev(b[2])
            l0 = ops.mf_bpr_loss(P, Q, ws, bu, bi, bj, hp).item()                 # calc_loss only
            loss = ops.mf_bpr_train_steps(P, Q, ws, bu, bi, bj, b.shape[1], 0, 1, hp, adam_step0=s).item()
            assert abs(l0 - losses[s]) <= 1e-5 * abs(losses[s]) and abs(loss - losses[s]) <= 1e-5 * abs(losses[s])
            tol = 2e-6 if opt == 0 else 2e-5
            for got, want in ((P, Ps[s + 1]), (Q, Qs[s + 1])):
                np.testing.assert_allclose(got.cpu().numpy(), want, rtol=0, atol=tol * max(1.0, np.abs(want).max()))


@pytest.mark.parametrize("F,B,opt", [(64, 4096, "sgd"), (32, 1000, "sgd"), (128, 777, "sgd"), (100, 513, "sgd"),
                                     (24, 300, "adam"), (7, 129, "sgd"), (256, 600, "sgd"), (1024, 300, "sgd"), (2, 64, "sgd")])
def test_mf_step_vs_oracle_random(ops, orc, F, B, opt):
    rng = np.random.default_rng(F * 1000 + B)
    U, I = 500, 300
    P0 = (rng.standard_normal((U, F)) * 0.3).astype(np.float32)
    Q0 = (rng.standard_normal((I, F)) * 0.3).astype(np.float32)
    hp_o, hp_d = orc.hyper(0.01, 0.002, 0.003, opt), ops.hyper(0.01, 0.002, 0.003, opt)
    Po, Qo = P0.copy(), Q0.copy()
    adam = None if opt == "sgd" else tuple(np.zeros_like(a) for a in (Po, Po, Qo, Qo))
    P, Q = dev(P0), dev(Q0)
    ws = ops.MFWorkspace(U, I, F, opt, "cuda")
    for s in range(3):
        b = np.stack([rng.integers(U, size=B), np.minimum(I - 1, rng.zipf(1.3, size=B) - 1),
                      rng.integers(I, size=B)]).astype(np.int32)
        lo, _ = orc.mf_bpr_step(Po, Qo, b[0].copy(), b[1].copy(), b[2].copy(), hp_o, True, adam, s + 1)
        ld = ops.mf_bpr_train_steps(P, Q, ws, dev(b[0]), dev(b[1]), dev(b[2]), B, 0, 1, hp_d, adam_step0=s).item()
        assert abs(ld - lo) <= 2e-6 * abs(lo)                    # loss: fp32 assembly of fp64 sums
        tol = 3e-6 if opt == "sgd" else 3e-5
        np.testing.assert_allclose(P.cpu().numpy(), Po, rtol=0, atol=tol)
        np.testing.assert_allclose(Q.cpu().numpy(), Qo, rtol=0, atol=tol)


def test_mf_epoch_ml100k_golden(ops):
    """BASELINE config 1 on the GPU: same init, triples and permutation as the reference run."""
    gs, gf = golden("ml100k_sampler"), golden("ml100k_fit")
    U, I, G, seed = (int(v) for v in gs["meta"])
    cu, ci = gs["coo_u"].astype(np.int32), gs["coo_i"].astype(np.int32)
    triples = np.stack([np.repeat(cu, G), np.repeat(ci, G), gs["triples_j"].astype(np.int32)], 1).astype(np.int32)
    lr, r1, r2, B, F = gf["hyper"]
    B, F = int(B), int(F)
    P, Q = dev(gf["P0"]), dev(gf["Q0"])
    bu, bi, bj = ops.gather_triples(dev(triples), dev(gf["perm"].astype(np.int64)))
    ws = ops.MFWorkspace(U, I, F, "sgd", "cuda")
    nsteps = (len(triples) + B - 1) // B
    losses = ops.mf_bpr_train_steps(P, Q, ws, bu, bi, bj, B, 0, nsteps, ops.hyper(lr, r1, r2)).cpu().numpy()
    ref = gf["step_losses"]
    assert nsteps == 1225 == len(ref)
    assert np.max(np.abs(losses - ref) / np.abs(ref)) < 2e-5
    assert abs(losses.sum() - ref.sum()) / ref.sum() < 1e-5       # north_star gate is 1e-4
    for got, want in ((P.cpu().numpy(), gf["P1"]), (Q.cpu().numpy(), gf["Q1"])):
        err = np.abs(got - want)
        assert err.max() < 1e-4 and (err < 5e-6).mean() > 0.999


def test_multi_step_launch_equals_single_steps(ops):
    rng = np.random.default_rng(9)
    U, I, F, B, n = 2000, 1500, 64, 2048, 2048 * 6 + 100
    P0 = (rng.standard_normal((U, F)) * 0.1).astype(np.float32)
    Q0 = (rng.standard_normal((I, F)) * 0.1).astype(np.float32)
    b = [dev(rng.integers(m, size=n).astype(np.int32)) for m in (U, I, I)]
    hp = ops.hyper(0.01, 0.001, 0.001)
    Pa, Qa, Pb, Qb = dev(P0), dev(Q0), dev(P0), dev(Q0)
    wa, wb = ops.MFWorkspace(U, I, F, "sgd", "cuda"), ops.MFWorkspace(U, I, F, "sgd", "cuda")
    la = ops.mf_bpr_train_steps(Pa, Qa, wa, *b, B, 0, 7, hp).cpu().numpy()
    lb = np.array([ops.mf_bpr_train_steps(Pb, Qb, wb, *b, B, s, 1, hp).item() for s in range(7)])
    np.testing.assert_allclose(la, lb, rtol=1e-6)
    np.testing.assert_allclose(Pa.cpu().numpy(), Pb.cpu().numpy(), atol=2e-6)
    np.testing.assert_allclose(Qa.cpu().numpy(), Qb.cpu().numpy(), atol=2e-6)


def test_nan_loss_raises_and_keeps_tables(ops):
    U, I, F, B = 50, 40, 32, 64
    P0 = np.full((U, F), 0.1, np.float32)
    P0[3, 5] = np.nan
    Q0 = np.full((I, F), 0.1, np.float32)
    P, Q = dev(P0), dev(Q0)
    b = [dev(np.full(B, 3, np.int32)), dev(np.arange(B, dtype=np.int32) % I), dev(np.zeros(B, np.int32))]
    ws = ops.MFWorkspace(U, I, F, "sgd", "cuda")
    with pytest.raises(ValueError):                               # AbstractRecommender.py:122-123
        ops.mf_bpr_train_steps(P, Q, ws, *b, B, 0, 1, ops.hyper(0.01, 0.001, 0.001))
    assert np.array_equal(Q.cpu().numpy(), Q0)                    # raised before backward/step


def test_host_step_entry_matches_device_entry(ops):
    rng = np.random.default_rng(10)
    U, I, F, B = 800, 600, 64, 3001
    P0 = (rng.standard_normal((U, F)) * 0.1).astype(np.float32)
    Q0 = (rng.standard_normal((I, F)) * 0.1).astype(np.float32)
    hb = [torch.from_numpy(rng.integers(m, size=B).astype(np.int32)).pin_memory() for m in (U, I, I)]
    hp = ops.hyper(0.01, 0.001, 0.001)
    Pa, Qa, Pb, Qb = dev(P0), dev(Q0), dev(P0), dev(Q0)
    wa, wb = ops.MFWorkspace(U, I, F, "sgd", "cuda"), ops.MFWorkspace(U, I, F, "sgd", "cuda")
    l_host = ops.mf_bpr_train_step_host(Pa, Qa, wa, *hb, hp, ops.stage_buffer(B, "cuda"))
    l_dev = ops.mf_bpr_train_steps(Pb, Qb, wb, *[t.cuda() for t in hb], B, 0, 1, hp).item()
    assert abs(l_host - l_dev) <= 1e-6 * abs(l_dev)
    np.testing.assert_allclose(Pa.cpu().numpy(), Pb.cpu().numpy(), atol=2e-6)


def test_fused_negative_sampling_mode(ops):
    """Throughput mode (sampler fused into the step): the drawn negatives lie in the complement of the user's row, are
    uniform over it, change per step, and a table-mode step on the SAME negatives reproduces the fused step."""
    rng = np.random.default_rng(21)
    U, I, F, B, nnz = 1200, 900, 64, 4096, 40_000
    cu = rng.integers(U, size=nnz).astype(np.int32)
    ci = np.minimum(I - 1, rng.zipf(1.2, size=nnz) - 1).astype(np.int32)
    row_ptr, col = csr_from_coo(cu, ci, U)
    P0 = (rng.standard_normal((U, F)) * 0.1).astype(np.float32)
    Q0 = (rng.standard_normal((I, F)) * 0.1).astype(np.float32)
    n = 3 * B
    sel = rng.integers(nnz, size=n)
    bu, bi = dev(cu[sel]), dev(ci[sel])
    neg = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    hp = ops.hyper(0.01, 0.001, 0.001)
    Pa, Qa = dev(P0), dev(Q0)
    wa = ops.MFWorkspace(U, I, F, "sgd", "cuda")
    la = ops.mf_bpr_train_steps_fused_neg(Pa, Qa, wa, bu, bi, dev(row_ptr), dev(col), 99, B, 0, 3, hp, neg_out=neg).cpu().numpy()
    j = neg.cpu().numpy()
    assert (j >= 0).all() and (j < I).all()
    pos = set(zip(cu.tolist(), ci.tolist()))
    assert not any((int(u), int(x)) in pos for u, x in zip(cu[sel], j))          # complement membership
    assert len(np.unique(j)) > 0.5 * min(I, n) and abs(j.mean() / I - 0.5) < 0.05   # spread over the item range
    # same (u, i) pair drawn in different steps gets different negatives (fresh per triple and step)
    neg2 = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    ops.mf_bpr_train_steps_fused_neg(dev(P0), dev(Q0), ops.MFWorkspace(U, I, F, "sgd", "cuda"), bu, bi, dev(row_ptr), dev(col), 100,
                                     B, 0, 3, hp, neg_out=neg2)
    assert (neg2 != neg).float().mean() > 0.9
    # equivalence: table mode on the recorded negatives
    Pb, Qb = dev(P0), dev(Q0)
    wb = ops.MFWorkspace(U, I, F, "sgd", "cuda")
    lb = ops.mf_bpr_train_steps(Pb, Qb, wb, bu, bi, neg, B, 0, 3, hp).cpu().numpy()
    np.testing.assert_allclose(la, lb, rtol=1e-6)
    np.testing.assert_allclose(Pa.cpu().numpy(), Pb.cpu().numpy(), atol=2e-6)
    np.testing.assert_allclose(Qa.cpu().numpy(), Qb.cpu().numpy(), atol=2e-6)


def test_pipelined_host_steps_match_device_steps(ops):
    rng = np.random.default_rng(12)
    U, I, F, B, n = 900, 700, 64, 2048, 2048 * 5 + 77
    P0 = (rng.standard_normal((U, F)) * 0.1).astype(np.float32)
    Q0 = (rng.standard_normal((I, F)) * 0.1).astype(np.float32)
    hb = [torch.from_numpy(rng.integers(m, size=n).astype(np.int32)).pin_memory() for m in (U, I, I)]
    hp = ops.hyper(0.01, 0.001, 0.001)
    Pa, Qa, Pb, Qb = dev(P0), dev(Q0), dev(P0), dev(Q0)
    wa, wb = ops.MFWorkspace(U, I, F, "sgd", "cuda"), ops.MFWorkspace(U, I, F, "sgd", "cuda")
    la = ops.mf_bpr_train_steps_host(Pa, Qa, wa, *hb, B, 6, hp).numpy()
    lb = ops.mf_bpr_train_steps(Pb, Qb, wb, *[t.cuda() for t in hb], B, 0, 6, hp).cpu().numpy()
    np.testing.assert_allclose(la, lb, rtol=1e-6)
    np.testing.assert_allclose(Pa.cpu().numpy(), Pb.cpu().numpy(), atol=2e-6)
    np.testing.assert_allclose(Qa.cpu().numpy(), Qb.cpu().numpy(), atol=2e-6)
    # NaN is sticky across the pipelined steps and surfaces as the reference's ValueError
    Pa[3, 3] = float("nan")
    with pytest.raises(ValueError):
        ops.mf_bpr_train_steps_host(Pa, Qa, wa, *hb, B, 6, hp)


# ------------------------------------------------------------------ rank / full_rank / predict
def test_mf_rank_golden(ops):
    g = golden("mf_rank")
    for c in range(int(g["ncases"])):
        P, Q = dev(g[f"c{c}_P"]), dev(g[f"c{c}_Q"])
        users, cands, K = g[f"c{c}_users"], g[f"c{c}_cands"].astype(np.int64), int(g[f"c{c}_K"])
        got = ops.mf_rank(P, Q, dev(users), dev(cands), K).cpu().numpy()
        assert got.dtype == np.float32 and np.array_equal(got, g[f"c{c}_preds"])
        full = ops.mf_full_rank(P, Q, dev(users[:5]), K).cpu().numpy()
        assert full.dtype == np.int64 and np.array_equal(full, g[f"c{c}_full"])
        assert np.array_equal(ops.mf_rank_host(P, Q, users, cands, K), g[f"c{c}_preds"])


def test_ml100k_rank_golden(ops):
    gf, gr = golden("ml100k_fit"), golden("ml100k_rank")
    P, Q, K = dev(gf["P1"]), dev(gf["Q1"]), int(gr["topk"])
    users, cands = gr["test_u"].astype(np.int64), gr["cands"].astype(np.int64)
    got = ops.mf_rank(P, Q, dev(users), dev(cands), K).cpu().numpy()
    assert np.array_equal(got, gr["preds"])
    assert np.array_equal(ops.mf_full_rank(P, Q, dev(users[:16]), K).cpu().numpy(), gr["full"])
    pp = ops.mf_predict(P, Q, dev(users[:8].astype(np.int32)), dev(cands[:8, -1].astype(np.int32))).cpu().numpy()
    np.testing.assert_allclose(pp, gr["pred_pairs"], rtol=2e-5, atol=1e-9)


@pytest.mark.parametrize("F,I,C,K", [(64, 5000, 1000, 50), (32, 9000, 1000, 50), (100, 700, 333, 20),
                                     (128, 12000, 4097, 100), (6, 100, 64, 64), (64, 30000, 1000, 50), (512, 3000, 700, 50), (1, 50, 20, 5)])
def test_rank_vs_oracle_bit_exact(ops, orc, F, I, C, K):
    rng = np.random.default_rng(F + I + C)
    U, n = 200, 37
    P = (rng.standard_normal((U, F)) * 0.2).astype(np.float32)
    Q = (rng.standard_normal((I, F)) * 0.2).astype(np.float32)
    Q[5] = Q[9]                                                   # exact score ties between distinct ids
    users = rng.integers(U, size=n).astype(np.int64)
    cands = rng.integers(I, size=(n, C)).astype(np.int64)
    cands[:, 1] = 5; cands[:, 0] = 9
    got = ops.mf_rank(dev(P), dev(Q), dev(users), dev(cands), K).cpu().numpy()
    assert np.array_equal(got, orc.mf_rank(P, Q, users, cands, K))
    gotf = ops.mf_full_rank(dev(P), dev(Q), dev(users[:6]), K).cpu().numpy()
    assert np.array_equal(gotf, orc.mf_full_rank(P, Q, users[:6], K))
    u32, i32 = users.astype(np.int32), cands[:, 0].astype(np.int32)
    assert np.array_equal(ops.mf_predict(dev(P), dev(Q), dev(u32), dev(i32)).cpu().numpy(), orc.mf_predict(P, Q, u32, i32))


def _topk_scores(rng, count, K):
    """score rows [9, count]: random; all equal; mixed +0.0 / -0.0 among +-1; four distinct values (long tie runs); a run of
    the row's best score straddling every chunk boundary of topk_scores_kernel (the key buffer of 4 096, then 4 096 - K new
    keys per chunk); ascending (every chunk replaces the running best); descending; the best score at both ends; a tie run at
    the K-th place"""
    S = rng.standard_normal((9, count)).astype(np.float32)
    S[1] = 0.75
    S[2] = rng.choice(np.array([-1.0, -0.0, 0.0, 1.0], np.float32), count)
    S[3] = rng.integers(0, 4, count)
    S[4] = -np.abs(S[4])
    for c in range(4096, count, 4096 - K) if count > 4096 else range(min(64, count - 1), count, 64):
        S[4, max(0, c - 40):c + 40] = 3.0
    S[5] = np.sort(S[5])
    S[6] = np.sort(S[6])[::-1]
    S[7, 0] = S[7, -1] = S[7].max() + 1
    srt = np.sort(S[8])[::-1]
    hi, lo = srt[max(0, K - 1 - K // 4)], srt[min(count - 1, K + K // 4)]
    S[8][(S[8] >= lo) & (S[8] <= hi)] = hi
    return S


@pytest.mark.parametrize("count", [1, 63, 64, 65, 4095, 4096, 4097, 8193, 26744])
def test_topk_from_scores_vs_stable_sort(ops, count):
    """drb_topk_from_scores (topk_scores_kernel: VAE, NeuMF and NFM scoring) bit for bit against a stable sort by score
    descending, then position ascending (+0.0 == -0.0), with candidate ids (float32 out, ids in [2^16, 2^24)) and without (int64
    positions), at K = 1, 50, 2 047 and 2 048 (K = count where count is smaller): one key buffer, and past it the chunks merged
    with the running best K"""
    rng = np.random.default_rng(count)
    for K in sorted({min(count, k) for k in (1, 50, 2047, 2048)}):
        S = _topk_scores(rng, count, K)
        pos = np.argsort(-S, axis=1, kind="stable")[:, :K]
        cands = rng.integers(1 << 16, 1 << 24, S.shape).astype(np.int64)
        cands[:, -1] = (1 << 24) - 1                             # the largest id a float32 holds exactly
        got_i = ops.topk_from_scores(dev(S), None, K).cpu().numpy()
        assert got_i.dtype == np.int64 and np.array_equal(got_i, pos), (count, K)
        got_f = ops.topk_from_scores(dev(S), dev(cands), K).cpu().numpy()
        want_f = np.take_along_axis(cands, pos, 1).astype(np.float32)
        assert got_f.dtype == np.float32 and np.array_equal(got_f, want_f), (count, K)


def test_topk_from_scores_refuses_bad_k(ops):
    from daisyrec_b200._lib import DrbError
    S = dev(np.zeros((2, 5000), np.float32))
    for K, cnt in ((2049, 5000), (11, 10)):
        for cands in (None, dev(np.zeros((2, cnt), np.int64))):
            with pytest.raises(DrbError, match="topk_from_scores: bad arguments"):
                ops.topk_from_scores(S[:, :cnt].contiguous(), cands, K)


# ------------------------------------------------------------------ the DataLoader's epoch order on the device
@pytest.mark.parametrize("n", [1, 2, 3, 5, 623, 624, 625, 1000, 4097, 100_003, 3_000_000])
def test_randperm_torch_is_bit_exact(n):
    """drb_randperm_torch == torch.randperm(n, generator=CPU generator seeded the same) for every n (MT19937 stream +
    parallel Fisher-Yates with deterministic reservations vs ATen's sequential walk)."""
    from daisyrec_b200 import ops
    for seed in (0, 2022, (1 << 40) + 17, (1 << 63) - 5):
        g = torch.Generator()
        g.manual_seed(seed)
        want = torch.randperm(n, generator=g)
        got = ops.randperm_torch(seed, n, "cuda").cpu()
        assert torch.equal(got, want), (n, seed)
        if n > 100_000:
            break


def test_mt19937_stream_matches_numpy():
    from daisyrec_b200 import ops
    for seed, n in ((5, 1), (7, 624), (11, 625), (2022, 200_000)):
        want = np.random.RandomState(seed).randint(0, 2 ** 32, size=n, dtype=np.uint64).astype(np.uint32)
        got = ops.mt19937_stream(seed, n, "cuda").cpu().numpy().view(np.uint32)
        assert np.array_equal(got, want), (seed, n)


def test_fit_shuffle_engines_agree():
    """shuffle_engine='torch' (permutation computed on the device) trains on exactly the batches of 'torch-cpu'
    (torch.randperm on the host generator): identical step order => bitwise-identical epoch losses are not guaranteed
    (atomics), but the permutation is, and the losses agree to fp32 accumulation noise."""
    import logging
    from daisyrec_b200.model import MF
    from daisyrec_b200.model.AbstractRecommender import epoch_permutation
    from daisyrec_b200.utils.dataset import BasicDataset, get_dataloader
    rng = np.random.default_rng(3)
    U, I, T = 300, 200, 50_000
    data = np.stack([rng.integers(U, size=T), rng.integers(I, size=T), rng.integers(I, size=T)], 1).astype(np.int32)
    tabs = {}
    for engine in ("torch", "torch-cpu"):
        cfg = dict(gpu="", logger=logging.getLogger("t"), lr=0.01, reg_1=0.001, reg_2=0.001, epochs=2, topk=10, user_num=U,
                   item_num=I, factors=32, loss_type="BPR", optimizer="default", init_method="default", early_stop=False,
                   progress=False, shuffle_engine=engine)
        torch.manual_seed(99)
        m = MF(cfg)
        m.fit(get_dataloader(BasicDataset(data), batch_size=1024, shuffle=True))
        tabs[engine] = (m.embed_user.weight.cpu().numpy(), m.embed_item.weight.cpu().numpy(), torch.get_rng_state())
    assert torch.equal(tabs["torch"][2], tabs["torch-cpu"][2])                  # the global RNG moved identically
    for a, b in zip(tabs["torch"][:2], tabs["torch-cpu"][:2]):
        # same batches => same tables up to atomic-order noise; an element that sits at ~0 may take the L1 term with the other
        # sign (sgn(theta) flips at 1e-9): lr * reg_1 * occurrences, on a handful of elements
        d = np.abs(a - b)
        assert (d > 5e-6).mean() < 2e-3 and d.max() < 1e-3, (float(d.max()), float((d > 5e-6).mean()))
    # and the device permutation itself equals the DataLoader protocol's
    from daisyrec_b200 import ops
    torch.manual_seed(5)
    want = epoch_permutation(T, True)
    torch.manual_seed(5)
    from daisyrec_b200.model.AbstractRecommender import epoch_seed
    assert torch.equal(ops.randperm_torch(epoch_seed(True), T, "cuda").cpu(), want)
