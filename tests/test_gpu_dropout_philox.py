"""NGCF and NFM with dropout_engine='philox': masks drawn inside the kernels from Philox, and NGCF's node dropout.

- the hooks' masks (drb_ngcf_philox_masks / drb_nfm_philox_masks, the kernels' own __device__ functions): kept fractions,
  independence across keys, and edges e / mirror(e) kept independently;
- the kernels use exactly those masks: a 'philox' forward equals the host-mask path fed the hook's bytes, bitwise on a graph
  whose adjacency rows all fit one SpMM segment (<= 256 edges, plain stores).  Steps are compared at the tolerance of the
  NGCF / NFM dropout checks of test_gpu_zzz_late.py: gradient accumulation in a step is not run-to-run deterministic -- the
  MF step kernel's phase 1 adds NGCF's representation gradient with RED.ADD, and nfm_head_bwd_kernel / nfm_scatter_kernel add
  NFM's bias and factor gradients with float atomics, in scheduling order;
- node dropout: the forward equals ngcf_forward on the explicitly dropped adjacency (bitwise), and one SGD step equals an fp64
  autograd restatement of the reference's forward() / calc_loss on the non-symmetric A_drop -- a restatement whose backward
  uses A_drop instead of A_drop^T is off by more than 10x the bound;
- class behaviour (steps_per_launch, the one seed draw per fit, eval mode, the engine key) and quality on the ml-100k split.
  The quality check is statistical: a fit sums its gradients in scheduling order, so even one engine and seed does not give
  the same KPIs twice; at larger NFM learning rates (0.01) single fits swing by more than 0.1 NDCG@10 either way.
"""
import logging

import numpy as np
import pytest
import torch

from conftest import golden

pytestmark = pytest.mark.gpu


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def graph_of(rng, U, I, nnz, hub=False):
    """-> (row_ptr, col, val) of A_hat over a random interaction set; hub: item 0 interacts with every user (rows > 256 edges)"""
    from daisyrec_b200 import ops
    cu, ci = rng.integers(U, size=nnz), rng.integers(I, size=nnz)
    if hub:
        cu, ci = np.concatenate([cu, np.arange(U)]), np.concatenate([ci, np.zeros(U, np.int64)])
    return ops.lgcn_norm_adj(cu, ci, U, I)


def within_6_sigma(kept, total, p):
    return abs(kept - (1 - p) * total) <= 6 * np.sqrt(total * p * (1 - p))


# ------------------------------------------------------------------ 1. mask statistics
@pytest.mark.parametrize("p", [0.1, 0.5])
def test_ngcf_mask_statistics(p):
    from daisyrec_b200 import ops
    rng = np.random.default_rng(1)
    U, I, dims = 1500, 2500, [16, 32, 32, 24]
    row_ptr, col, val = graph_of(rng, U, I, 40000)
    graph = ops.LgcnGraph(row_ptr, col, val, "cuda")
    nnz, n = len(col), U + I
    keep, edge = ops.ngcf_philox_masks(7, 3, U, I, dims, p, p, nnz, "cuda")
    keep, edge = keep.cpu().numpy(), edge.cpu().numpy()
    assert set(np.unique(keep)) <= {0, 1} and set(np.unique(edge)) <= {0, 1}
    off = 0
    layers = []
    for w in dims[1:]:
        blk = keep[off:off + n * w]
        assert within_6_sigma(int(blk.sum()), blk.size, p), (p, w)
        layers.append(blk)
        off += n * w
    assert within_6_sigma(int(edge.sum()), nnz, p)
    assert not np.array_equal(layers[1], layers[2])                    # layers 1 and 2 have the same width: different masks
    for other in ((8, 3), (7, 4)):                                     # another seed, another forward
        k2, e2 = ops.ngcf_philox_masks(*other, U, I, dims, p, p, nnz, "cuda")
        assert (k2.cpu().numpy() != keep).mean() > 0.5 * 2 * p * (1 - p)
        assert (e2.cpu().numpy() != edge).mean() > 0.5 * 2 * p * (1 - p)
    # e and mirror(e): kept together at rate k^2 (the two directions of an interaction are independent entries)
    mirror = graph.edge_mirror()[:nnz].cpu().numpy()
    r = np.repeat(np.arange(n), np.diff(row_ptr))
    assert np.array_equal(r[mirror], col) and np.array_equal(col[mirror], r) and np.array_equal(mirror[mirror], np.arange(nnz))
    half = r < col                                                     # one slot per pair
    both = int((edge[half] & edge[mirror[half]]).sum())
    assert within_6_sigma(both, int(half.sum()), 1 - (1 - p) ** 2), (both, int(half.sum()))
    k0, e0 = ops.ngcf_philox_masks(7, 3, U, I, dims, 0.0, 0.0, nnz, "cuda")
    assert bool(k0.all()) and bool(e0.all())


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_nfm_mask_statistics(p):
    from daisyrec_b200 import ops
    B, F, L = 4096, 24, 2
    m = ops.nfm_philox_masks(11, 5, B, F, L, p, "cuda").cpu().numpy().reshape(2, 1 + L, B, F)
    assert within_6_sigma(int(m.sum()), m.size, p)
    for side in range(2):
        for site in range(1 + L):
            assert within_6_sigma(int(m[side, site].sum()), B * F, p)
    assert not np.array_equal(m[0], m[1])                              # pos and neg calls
    assert not np.array_equal(m[0, 0], m[0, 1])                        # sites
    for other in ((12, 5), (11, 6)):                                   # seeds, steps
        m2 = ops.nfm_philox_masks(*other, B, F, L, p, "cuda").cpu().numpy().reshape(m.shape)
        assert (m2 != m).mean() > 0.5 * 2 * p * (1 - p)
    assert bool(ops.nfm_philox_masks(11, 5, B, F, L, 0.0, "cuda").all())


# ------------------------------------------------------------------ 2. the kernels use the hooks' masks
def _ngcf_setup(seed=3, U=200, I=300, nnz=3000, dims=(16, 32, 24), hub=False):
    from daisyrec_b200 import ops
    rng = np.random.default_rng(seed)
    row_ptr, col, val = graph_of(rng, U, I, nnz, hub)
    E = (rng.standard_normal((U + I, dims[0])) * 0.1).astype(np.float32)
    W = (rng.standard_normal(ops.ngcf_param_count(list(dims))) * 0.1).astype(np.float32)
    return rng, (row_ptr, col, val), E, W, list(dims)


def assert_step_close(runs, lr, opt, tol_sgd, what):
    """[losses, tensors...] of the philox run and of the host-mask run: losses within 3e-5, tensors within the late checks'
    bound (99 % of elements within tol, none beyond the 2 lr an Adam step on a ~0 gradient can take)"""
    a, c = runs
    np.testing.assert_allclose(a[0], c[0], rtol=3e-5, atol=0, err_msg=what)
    for k, (got, want) in enumerate(zip(a[1:], c[1:])):
        if want.size == 0:
            continue
        err = np.abs(got - want)
        tol = (tol_sgd if opt == "sgd" else 10 * tol_sgd) * max(1.0, np.abs(want).max())
        assert (err <= tol).mean() >= 0.99 and err.max() <= 2.1 * lr + tol, (what, k, float((err <= tol).mean()), float(err.max()))


def test_ngcf_message_dropout_matches_host_masks():
    from daisyrec_b200 import ops
    rng, (row_ptr, col, val), E_h, W_h, dims = _ngcf_setup()
    assert np.diff(row_ptr).max() <= 256
    U, I = 200, 300
    graph = ops.LgcnGraph(row_ptr, col, val, "cuda")
    B, S, p, seed, f0 = 512, 3, 0.1, 99, 17
    b = [dev(rng.integers(n, size=B * S).astype(np.int32)) for n in (U, I, I)]
    keeps = [ops.ngcf_philox_masks(seed, f0 + s, U, I, dims, p, 0.0, 0, "cuda")[0] for s in range(S)]
    for opt in ("sgd", "adam"):
        hp = ops.hyper(0.05, 1e-3, 1e-3, opt)
        runs = []
        for host in (False, True):
            E, W = dev(E_h), dev(W_h)
            ws = ops.NgcfWorkspace(U, I, dims, opt, "cuda")
            if host:
                loss = ops.ngcf_bpr_train_steps(E, W, ws, graph, *b, B, 0, S, hp, dropout=p, keep=torch.cat(keeps))
            else:
                loss = ops.ngcf_bpr_train_steps_philox(E, W, ws, graph, *b, B, 0, S, hp, seed=seed, forward0=f0, mess_dropout=p)
            runs.append([loss.cpu().numpy(), E.cpu().numpy(), W.cpu().numpy()])
        assert runs[0][0][0] == runs[1][0][0], opt                     # the first step's loss: same forward, same masks
        assert_step_close(runs, 0.05, opt, 5e-6, f"ngcf {opt}")
    ws = ops.NgcfWorkspace(U, I, dims, "sgd", "cuda")
    E, W = dev(E_h), dev(W_h)
    got = ops.ngcf_forward_philox(E, W, ws, graph, seed=seed, forward=f0 + 1, mess_dropout=p).cpu().numpy()
    want = ops.ngcf_forward(E, W, ws, graph, dropout=p, keep=keeps[1]).cpu().numpy()
    assert np.array_equal(got, want)
    plain = ops.ngcf_forward(E, W, ws, graph).cpu().numpy()
    assert not np.array_equal(got, plain)


def test_nfm_dropout_matches_host_masks():
    from daisyrec_b200 import ops
    rng = np.random.default_rng(5)
    U, I, F, L, B, S, p, seed = 300, 400, 32, 2, 1024, 3, 0.5, 1234
    for bn, act, opt in ((True, 0, "sgd"), (False, 2, "adam")):
        P_h = (rng.standard_normal((U, F)) * 0.1).astype(np.float32)
        Q_h = (rng.standard_normal((I, F)) * 0.1).astype(np.float32)
        bias_h = (rng.standard_normal(U + I + 1) * 0.01).astype(np.float32)
        N_h = (rng.standard_normal(ops.nfm_param_count(F, L, bn)) * 0.2).astype(np.float32)
        R_h = np.tile(np.concatenate([np.zeros(F), np.ones(F)]).astype(np.float32), 1 + L) if bn else np.zeros(0, np.float32)
        b = [dev(rng.integers(n, size=B * S).astype(np.int32)) for n in (U, I, I)]
        hp = ops.hyper(0.05, 1e-3, 1e-3, opt)
        step0 = 4
        keep = torch.cat([ops.nfm_philox_masks(seed, step0 + s, B, F, L, p, "cuda") for s in range(S)])
        runs = []
        for host in (False, True):
            ts = [dev(x) for x in (P_h, Q_h, bias_h, N_h, R_h)]
            ws = ops.NfmWorkspace(U, I, F, L, bn, opt, 2 * B, "cuda")
            args = (*ts, ws, act, *b, B, 0, S, hp)
            if host:
                loss = ops.nfm_bpr_train_steps(*args, adam_step0=step0, dropout=p, keep=keep)
            else:
                loss = ops.nfm_bpr_train_steps_philox(*args, adam_step0=step0, dropout=p, seed=seed)
            runs.append([loss.cpu().numpy()] + [t.cpu().numpy() for t in ts])
        assert runs[0][0][0] == runs[1][0][0], (bn, act, opt)
        assert_step_close(runs, 0.05, opt, 1e-5, f"nfm bn={bn} act={act} {opt}")


# ------------------------------------------------------------------ 3. node-dropout forward
def _dropped_graph(row_ptr, col, val, edge, p):
    inv = np.float32(1.0 / (1.0 - p))
    return np.where(edge.astype(bool), val * inv, np.float32(0)).astype(np.float32)


def test_ngcf_node_dropout_forward_equals_dropped_adjacency():
    from daisyrec_b200 import ops
    rng, (row_ptr, col, val), E_h, W_h, dims = _ngcf_setup(seed=4)
    U, I = 200, 300
    assert np.diff(row_ptr).max() <= 256
    graph = ops.LgcnGraph(row_ptr, col, val, "cuda")
    ws = ops.NgcfWorkspace(U, I, dims, "sgd", "cuda")
    E, W = dev(E_h), dev(W_h)
    for mess, node in ((0.1, 0.2), (0.0, 0.5)):
        keep, edge = ops.ngcf_philox_masks(21, 8, U, I, dims, mess, node, len(col), "cuda")
        got = ops.ngcf_forward_philox(E, W, ws, graph, seed=21, forward=8, mess_dropout=mess, node_dropout=node).cpu().numpy()
        dropped = ops.LgcnGraph(row_ptr, col, _dropped_graph(row_ptr, col, val, edge.cpu().numpy(), node), "cuda")
        want = ops.ngcf_forward(E, W, ws, dropped, dropout=mess, keep=keep if mess > 0 else None).cpu().numpy()
        assert np.array_equal(got, want), (mess, node)


# ------------------------------------------------------------------ 4. node-dropout backward against fp64 autograd
class _Spmm(torch.autograd.Function):
    """Y = A X with the backward dX = B^T dY: B = A is the true gradient, B = A^T the defect that treats A_drop as symmetric."""

    @staticmethod
    def forward(ctx, A, B, X):
        ctx.save_for_backward(B)
        return A @ X

    @staticmethod
    def backward(ctx, g):
        (B,) = ctx.saved_tensors
        return None, None, B.t() @ g


def ngcf_sgd_ref(E0, W, dims, A, keeps, scale, U, bu, bi, bj, lr, transpose_ok=True):
    """One SGD step of the reference's forward() / calc_loss (BPR, no regulariser) in fp64 with autograd -> (E0', W')"""
    E0 = torch.tensor(E0, dtype=torch.float64, requires_grad=True)
    Wt = torch.tensor(W, dtype=torch.float64, requires_grad=True)
    A = torch.tensor(A, dtype=torch.float64)
    B = A if transpose_ok else A.t()
    reps, E, o = [E0], E0, 0
    for l in range(len(dims) - 1):
        i, j = dims[l], dims[l + 1]
        W1 = Wt[o:o + i * j].view(j, i); o += i * j
        b1 = Wt[o:o + j]; o += j
        W2 = Wt[o:o + i * j].view(j, i); o += i * j
        b2 = Wt[o:o + j]; o += j
        X = _Spmm.apply(A, B, E)
        Y = ((E + X) @ W1.t() + b1) + ((X * E) @ W2.t() + b2)
        Z = torch.nn.functional.leaky_relu(Y, 0.2)
        if keeps is not None:
            Z = Z * torch.tensor(keeps[l], dtype=torch.float64) * scale
        E = torch.nn.functional.normalize(Z, p=2, dim=1)
        reps.append(E)
    R = torch.cat(reps, 1)
    x = (R[bu] * R[U + bi]).sum(1) - (R[bu] * R[U + bj]).sum(1)
    loss = -torch.log(1e-10 + torch.sigmoid(x)).sum()
    loss.backward()
    with torch.no_grad():
        return (E0 - lr * E0.grad).numpy(), (Wt - lr * Wt.grad).numpy()


@pytest.mark.parametrize("shape", ["unequal_widths", "long_rows"])
def test_ngcf_node_dropout_step_against_fp64(shape):
    from daisyrec_b200 import ops
    if shape == "unequal_widths":
        rng, (row_ptr, col, val), E_h, W_h, dims = _ngcf_setup(seed=6, dims=(24, 40, 16, 32))
    else:
        rng, (row_ptr, col, val), E_h, W_h, dims = _ngcf_setup(seed=7, U=400, I=300, nnz=4000, dims=(32, 32, 32), hub=True)
        assert np.diff(row_ptr).max() > 256
    U, I = (200, 300) if shape == "unequal_widths" else (400, 300)
    n, nnz = U + I, len(col)
    graph = ops.LgcnGraph(row_ptr, col, val, "cuda")
    B, lr, mess, node, seed, fwd = 2048, 0.05, 0.1, 0.3, 5, 2
    b = [rng.integers(m, size=B).astype(np.int32) for m in (U, I, I)]
    E, W = dev(E_h), dev(W_h)
    ws = ops.NgcfWorkspace(U, I, dims, "sgd", "cuda")
    ops.ngcf_bpr_train_steps_philox(E, W, ws, graph, *[dev(x) for x in b], B, 0, 1, ops.hyper(lr, 0.0, 0.0), seed=seed,
                                    forward0=fwd, mess_dropout=mess, node_dropout=node)
    keep, edge = ops.ngcf_philox_masks(seed, fwd, U, I, dims, mess, node, nnz, "cuda")
    keep = keep.cpu().numpy()
    keeps, off = [], 0
    for w in dims[1:]:
        keeps.append(keep[off:off + n * w].reshape(n, w))
        off += n * w
    A = np.zeros((n, n), np.float32)
    A[np.repeat(np.arange(n), np.diff(row_ptr)), col] = _dropped_graph(row_ptr, col, val, edge.cpu().numpy(), node)
    assert not np.array_equal(A, A.T)
    scale = float(np.float32(1.0) / np.float32(1.0 - np.float32(mess)))
    got = (E.cpu().numpy(), W.cpu().numpy())
    want = ngcf_sgd_ref(E_h, W_h, dims, A, keeps, scale, U, b[0], b[1], b[2], lr)
    wrong = ngcf_sgd_ref(E_h, W_h, dims, A, keeps, scale, U, b[0], b[1], b[2], lr, transpose_ok=False)
    worst_wrong = 0.0
    for g_, w_, x_, nm in zip(got, want, wrong, ("E0", "W")):
        tol = 5e-6 * max(1.0, np.abs(w_).max())                       # test_gpu_ngcf.py's bound on the SGD step
        err = np.abs(g_ - w_).max()
        assert err <= tol, (shape, nm, float(err), tol)
        worst_wrong = max(worst_wrong, np.abs(x_ - w_).max() / tol)
    assert worst_wrong > 10, (shape, worst_wrong)


# ------------------------------------------------------------------ 5. class behaviour
def _ngcf_cfg(U, I, coo_u, coo_i, **over):
    import pandas as pd
    from daisyrec_b200.utils.utils import get_inter_matrix
    df = pd.DataFrame({"user": coo_u, "item": coo_i, "rating": 1.0, "timestamp": np.arange(len(coo_u))})
    cfg = dict(gpu="", logger=logging.getLogger("t"), epochs=2, lr=0.01, reg_1=0.0, reg_2=1e-4, user_num=U, item_num=I,
               factors=16, hidden_size_list=[32, 16], node_dropout=0.0, mess_dropout=0.0, loss_type="BPR", optimizer="default",
               init_method="default", early_stop=False, topk=10, progress=False, UID_NAME="user", IID_NAME="item",
               INTER_NAME="rating", dropout_engine="philox")
    cfg["inter_matrix"] = get_inter_matrix(df, cfg)
    cfg.update(over)
    return cfg


def _nfm_cfg(U, I, **over):
    cfg = dict(gpu="", logger=logging.getLogger("t"), epochs=2, lr=0.01, reg_1=0.0, reg_2=0.0, user_num=U, item_num=I, factors=16,
               num_layers=2, batch_norm=True, act_function="relu", dropout=0.5, loss_type="BPR", optimizer="default",
               init_method="default", early_stop=False, topk=10, progress=False, dropout_engine="philox")
    cfg.update(over)
    return cfg


def _small_rows(seed=9, U=200, I=300, T=6000):
    rng = np.random.default_rng(seed)
    cu, ci = rng.integers(U, size=T // 2), rng.integers(I, size=T // 2)
    rows = np.stack([np.concatenate([cu, cu]), np.concatenate([ci, ci]), rng.integers(I, size=T)], 1).astype(np.int32)
    return cu, ci, rows


def _fit_losses(model, loader):
    rec = []
    orig = model._train_steps

    def wrap(*a):
        out = orig(*a)
        rec.append(out.cpu().numpy().copy())
        return out
    model._train_steps = wrap
    model.fit(loader)
    return np.concatenate(rec)


@pytest.mark.parametrize("model", ["ngcf", "nfm"])
def test_steps_per_launch_and_one_seed_draw(model):
    from daisyrec_b200.model import NFM, NGCF
    from daisyrec_b200.utils.dataset import BasicDataset, get_dataloader
    U, I = 200, 300
    cu, ci, rows = _small_rows()

    def make(**over):
        if model == "ngcf":
            return NGCF(_ngcf_cfg(U, I, cu, ci, **over))
        return NFM(_nfm_cfg(U, I, **over))
    drop = dict(mess_dropout=0.1, node_dropout=0.2) if model == "ngcf" else dict(dropout=0.5)
    nodrop = dict(mess_dropout=0.0, node_dropout=0.0) if model == "ngcf" else dict(dropout=0.0)
    runs, states = [], []
    for over in (dict(drop), dict(drop, steps_per_launch=1), dict(nodrop)):
        torch.manual_seed(3)
        m = make(**over)
        runs.append(_fit_losses(m, get_dataloader(BasicDataset(rows), batch_size=512, shuffle=True)))
        states.append(torch.get_rng_state())
    assert len(runs[0]) == len(runs[1]) == 2 * 12 and runs[0][0] == runs[1][0]
    np.testing.assert_allclose(runs[0], runs[1], rtol=3e-5, atol=0)    # step gradients are summed in scheduling order
    assert torch.equal(states[0], states[1])
    torch.set_rng_state(states[2])
    torch.empty((), dtype=torch.int64).random_()                      # the one seed draw of a 'philox' fit
    assert torch.equal(torch.get_rng_state(), states[0])


def test_ngcf_eval_mode_forward_and_engine_key():
    from daisyrec_b200.model import NFM, NGCF
    U, I = 200, 300
    cu, ci, _ = _small_rows()
    outs = {}
    for node, mess in ((0.5, 0.1), (0.0, 0.1), (0.0, 0.0)):
        torch.manual_seed(4)
        m = NGCF(_ngcf_cfg(U, I, cu, ci, node_dropout=node, mess_dropout=mess))
        m.eval()
        outs[(node, mess)] = torch.cat(m.forward()).cpu().numpy()
        if node > 0:
            m.train()
            assert not np.array_equal(torch.cat(m.forward()).cpu().numpy(), outs[(node, mess)])
    assert np.array_equal(outs[(0.5, 0.1)], outs[(0.0, 0.1)])          # SparseDropout is the identity in eval mode
    assert not np.array_equal(outs[(0.0, 0.1)], outs[(0.0, 0.0)])      # message dropout stays on
    for cls, cfg in ((NGCF, _ngcf_cfg(U, I, cu, ci)), (NFM, _nfm_cfg(U, I))):
        with pytest.raises(ValueError):
            cls(dict(cfg, dropout_engine="cudnn"))
    with pytest.raises(ValueError):
        NGCF(_ngcf_cfg(U, I, cu, ci, node_dropout=1.0))
    with pytest.raises(NotImplementedError):                           # host-parity node dropout stays refused
        NGCF(_ngcf_cfg(U, I, cu, ci, node_dropout=0.1, dropout_engine="torch"))


# ------------------------------------------------------------------ 6. quality on the ml-100k split
def _ml100k_split():
    gs, gr, gv = golden("ml100k_sampler"), golden("ml100k_rank"), golden("vae")
    U, I = (int(x) for x in gv["ml_meta"][:2])
    cu, ci = gs["coo_u"].astype(np.int64), gs["coo_i"].astype(np.int64)
    ng = len(gs["triples_j"]) // len(cu)
    rows = np.stack([np.repeat(cu, ng), np.repeat(ci, ng), gs["triples_j"].astype(np.int64)], 1).astype(np.int32)
    off = np.concatenate([[0], np.cumsum(gr["gt_len"])])
    gt = [set(gr["gt_flat"][off[k]:off[k + 1]].tolist()) for k in range(len(gr["test_u"]))]
    return U, I, cu, ci, rows, gr["test_u"].astype(np.int64), gr["cands"].astype(np.int64), gt


def _kpis(top, gt, k=10):
    rec, ndcg = [], []
    for row, g in zip(top, gt):
        hits = [1.0 if int(x) in g else 0.0 for x in row[:k]]
        rec.append(sum(hits) / len(g))
        idcg = sum(1.0 / np.log2(r + 2) for r in range(min(len(g), k)))
        ndcg.append(sum(h / np.log2(r + 2) for r, h in enumerate(hits)) / idcg)
    return float(np.mean(ndcg)), float(np.mean(rec))


@pytest.mark.parametrize("model", ["ngcf", "nfm"])
def test_quality_philox_within_torch_spread(model):
    from daisyrec_b200.model import NFM, NGCF
    from daisyrec_b200.utils.dataset import BasicDataset, CandidatesDataset, get_dataloader
    U, I, cu, ci, rows, test_u, cands, gt = _ml100k_split()
    res = {}
    for engine in ("torch", "philox"):
        for seed in (0, 1, 2):
            torch.manual_seed(seed)
            if model == "ngcf":
                m = NGCF(_ngcf_cfg(U, I, cu, ci, epochs=5, lr=0.01, factors=64, hidden_size_list=[64, 64], mess_dropout=0.1,
                                   dropout_engine=engine, topk=10))
            else:
                m = NFM(_nfm_cfg(U, I, epochs=5, lr=0.0005, factors=64, dropout=0.5, dropout_engine=engine, topk=10))
            m.fit(get_dataloader(BasicDataset(rows), batch_size=4096, shuffle=True))
            loader = get_dataloader(CandidatesDataset([[int(u), cands[r]] for r, u in enumerate(test_u)]), batch_size=128,
                                    shuffle=False)
            res[(engine, seed)] = _kpis(m.rank(loader), gt)
    print(model, {k: [round(x, 4) for x in v] for k, v in res.items()})
    for k, name in enumerate(("NDCG@10", "Recall@10")):
        t = [res[("torch", s)][k] for s in range(3)]
        lo, hi = min(t), max(t)
        w = hi - lo
        for s in range(3):
            v = res[("philox", s)][k]
            assert lo - w <= v <= hi + w, (model, name, v, t)
