"""NGCF + BPR steps with dropout against the float64 reference of test_gpu_graph_fp64.py (ngcf_ref with its masks), one
teacher-forced step at a time (fp64_step.py: the snapshot, the bound and its checks).

Masks.  dropout_engine 'philox': the bytes of ops.ngcf_philox_masks (the kernels' own keep functions) at the step's forward
counter; 'torch': message masks drawn here and fed to ngcf_bpr_train_steps.  The reference takes them as given, so they add
no P_e term: message dropout is z * keep * (1.0f / (float)(1 - p)) after the LeakyReLU (one more fp32 product per kept
element, carried by N_e) and the same factor on the fp32 dz of the normalise backward; node dropout is the forward over
A_drop (kept slots val * (float)(1 / (1 - p)), dropped slots 0, one edge mask for every layer of a forward) and the backward
AdX over A_drop^T, the noise chains over the same matrices.

Kernels under test: spmm_seg_drop_kernel (DROP 1 the forward, DROP 2 the backward through the mirror index), ngcf_mirror_kernel,
the message factor in ngcf_act_kernel / ngcf_act_bwd_kernel (the backward regenerates the mask), and the forward counter
forward0 + s of a multi-step launch.

KAPPA and PHI_FRAC_MAX are test_gpu_graph_fp64.py's (3 for the fp32 and the bf16 tower, 0.4); no case needs more.  Measured on
one H100 80GB HBM3 (700 W power limit); the GPU part of this file runs in about 60 s there.  "Needed" as in
test_gpu_graph_fp64.py: the per-element KAPPA of an SGD step where P_e = 0, else the smallest KAPPA of KAPPA_LADDER (from
0.125) at which every element of the step passes.
  Bench shape, Adam: 'philox' fp32 0.82, bf16 1.00 (elements that need P_e; at most 17 % of the intermediates flagged),
    'torch' fp32 0.77; kappa needed 0.125 on every step.  The forward with the same masks: 0.54 / 0.995, kappa needed 2
    (1.5 without dropout).
  Segment edges: fp32 <= 0.46, kappa needed 0.125; bf16 0.96 / 1.00 (node 0.1 / 0.5), kappa needed 0.25 / 0.5, at most 13 %
    flagged.
  Widths (mess 0.3 + node 0.2): fp32 <= 0.48, kappa needed 0.125; bf16 <= 0.97, kappa needed <= 0.5, at most 15 % flagged.
  Launches: singles <= 0.44 (fp32) / 0.44 (bf16); the 3-step launch within 0.006 / 0.17 of the singles' summed bound.
  Forward (ngcf_forward_philox, random graph): fp32 <= 0.36, bf16 <= 0.98, kappa needed <= 1.5.
A DROP 2 that reads the keep at slot e instead of mirror[e] (A_drop in place of A_drop^T) fails every step case with node
dropout here, at 1.9e6 - 8.2e9 x the bound.

The CPU tests show the bound sees dropout defects: a stand-in that multiplies the backward by A_drop instead of A_drop^T, draws
an edge mask per layer, leaves kept edges unscaled, skips the message factor in the backward, or runs step s on the masks of
forward s - 1, fails it (test_harness_flags_dropout_defect prints each ratio).
"""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)
from fp64_step import checked_step, launch_vs_singles, report, summary  # noqa: E402
from test_gpu_graph_fp64 import (NGCF_WIDTHS, Gpu, RefGraph, StandIn, _cpu_case, amazon_book, crafted_graph,  # noqa: E402
                                 ngcf_forward_check, planes_uniform, random_graph)


class DropGpu(Gpu):
    """NGCF steps with dropout through ops: engine 'philox' runs ngcf_bpr_train_steps_philox (step s of a launch at forward
    counter forward0 + s), 'torch' runs ngcf_bpr_train_steps with the message keep bytes of the step (message dropout only).
    masks(forward) -> one step's inputs for checked_step: keep, p, edge, node_p, forward."""

    def __init__(self, *args, engine="philox", seed=0, forward0=0, mess=0.0, node=0.0, gen=None, **kw):
        super().__init__(*args, **kw)
        assert engine == "philox" or node == 0.0
        self.engine, self.seed, self.forward0, self.mess, self.node, self.gen = engine, seed, forward0, mess, node, gen
        self.nnz = int(self.graph.col.numel())

    def masks(self, forward):
        n = self.U + self.I
        if self.engine == "philox":
            keep, edge = self.ops.ngcf_philox_masks(self.seed, forward, self.U, self.I, self.dims, self.mess, self.node, self.nnz,
                                                    "cuda")
        else:
            keep = (torch.rand(n * sum(self.dims[1:]), generator=self.gen, device="cuda") >= self.mess).to(torch.uint8)
            edge = None
        return dict(keep=keep if self.mess > 0 else None, p=self.mess, edge=edge if self.node > 0 else None, node_p=self.node,
                    forward=forward)

    def run(self, lo, n, batch, k, adam_step0=0, apply=True, first_step=0, keep=None, p=None, edge=None, node_p=None,
            forward=None):
        """without step inputs (a multi-step launch): the launch's own masks from forward0 ('philox')"""
        bu, bi, bj = (x[lo:lo + n] for x in self.planes)
        args = (self.t["E0"], self.t["W"], self.ws, self.graph, bu, bi, bj, batch, first_step, k, self.hp)
        mess = self.mess if p is None else p
        if self.engine == "philox":
            out = self.ops.ngcf_bpr_train_steps_philox(*args, adam_step0=adam_step0, apply=apply, tower_dtype=self.td,
                                                       seed=self.seed, forward0=self.forward0 if forward is None else forward,
                                                       mess_dropout=mess, node_dropout=self.node if node_p is None else node_p)
        else:
            assert k == 1 and keep is not None
            out = self.ops.ngcf_bpr_train_steps(*args, adam_step0=adam_step0, apply=apply, tower_dtype=self.td, dropout=mess,
                                                keep=keep)
        torch.cuda.synchronize()
        return out.cpu().numpy()


@pytest.fixture(scope="module")
def gpu():
    from daisyrec_b200 import ops
    ops.require_cuda()
    return ops


def _tables(ops, rng, U, I, dims):
    E0 = torch.from_numpy((rng.standard_normal((U + I, dims[0])) * 0.1).astype(np.float32)).cuda()
    W = torch.from_numpy((rng.standard_normal(ops.ngcf_param_count(dims)) * 0.15).astype(np.float32)).cuda()
    return E0, W


def _sgd_then_adam(make, B, tag, forward0):
    """one SGD step, then two Adam steps from the same start, each on its own forward's masks -> records"""
    st = make("sgd", 0.05)
    recs = [checked_step(st, 0, B, B, f"{tag} sgd", ref_device="cuda", **st.masks(forward0))]
    st = make("adam", 0.001)
    recs += [checked_step(st, s * B, B, B, f"{tag} adam {s}", adam_step0=s, ref_device="cuda", **st.masks(forward0 + 1 + s))
             for s in range(2)]
    return recs


# ---------------------------------------------------------------- GPU: the bench shape
@pytest.mark.gpu
@pytest.mark.parametrize("engine,td", [("philox", 0), ("philox", 1), ("torch", 0)])
def test_ngcf_dropout_bench_shape(gpu, engine, td):
    """bench_dropout's NGCF rows: Amazon-Book, widths 64/64/64/64, B = 65 536, Adam lr 0.001, reg (0, 1e-3); 'philox' with
    mess 0.1 + node 0.1 (rows of thousands of edges: many segments per row), 'torch' with mess 0.1; two checked steps.
    'philox' also checks the forward with the same masks."""
    ops = gpu
    B, dims = 65536, [64, 64, 64, 64]
    U, I, graph, rg, planes, g = amazon_book(B, 2, seed=31 + td)
    E0 = (torch.randn(U + I, 64, device="cuda", generator=g) * 0.05).contiguous()
    W = (torch.randn(ops.ngcf_param_count(dims), device="cuda", generator=g) * 0.1).contiguous()
    node = 0.1 if engine == "philox" else 0.0
    st = DropGpu(graph, rg, U, I, E0, W, planes, 3, "adam", 0.001, (0.0, 1e-3), dims, td, engine=engine, seed=2024,
                 forward0=40, mess=0.1, node=node, gen=g)
    recs = []
    if engine == "philox":
        m = st.masks(77)
        ws = ops.NgcfWorkspace(U, I, dims, "sgd", "cuda")
        got = ops.ngcf_forward_philox(E0, W, ws, graph, tower_dtype=td, seed=2024, forward=77, mess_dropout=0.1, node_dropout=node)
        r, need = ngcf_forward_check(ops, graph, rg, U, I, E0, W, dims, td, m["keep"], 0.1, m["edge"], node, got=got)
        print(f"forward philox td={td}: worst error/bound {r:.3g}, kappa needed {need:.3g}")
        assert r <= 1, r
    recs += [checked_step(st, s * B, B, B, f"{engine} td={td} adam {s}", adam_step0=s, ref_device="cuda", **st.masks(40 + s))
             for s in range(2)]
    report(f"ngcf dropout bench {engine} td={td}", recs)


# ---------------------------------------------------------------- GPU: segment edges
@pytest.mark.gpu
@pytest.mark.parametrize("td", [0, 1])
@pytest.mark.parametrize("node", [0.1, 0.5])
def test_ngcf_node_dropout_segment_edges(gpu, node, td):
    """rows of degree 0, 1, 3 - 5, 255 - 257, 511 - 513 and 4 099: DROP 1's Philox word cache across segment starts that are
    not multiples of 4, DROP 2's mirror read in the tail loop, multi-segment rows summed with red_row"""
    ops = gpu
    rng = np.random.default_rng(int(node * 10) + 3 * td)
    U, I, adj = crafted_graph(rng)
    graph, rg = ops.LgcnGraph(*adj, "cuda"), RefGraph(*adj, "cuda")
    dims = [64, 64, 32]
    E0, W = _tables(ops, rng, U, I, dims)
    B = 3000
    planes = planes_uniform(rng, U, I, 2 * B)

    def make(opt, lr):
        return DropGpu(graph, rg, U, I, E0, W, planes, 2, opt, lr, (1e-3, 1e-3), dims, td, seed=71, mess=0.1, node=node)
    report(f"ngcf segment edges node={node} td={td}", _sgd_then_adam(make, B, f"node={node} td={td}", 3))


# ---------------------------------------------------------------- GPU: layer widths
@pytest.mark.gpu
@pytest.mark.parametrize("td", [0, 1])
@pytest.mark.parametrize("dims", NGCF_WIDTHS, ids=lambda d: "-".join(map(str, d)))
def test_ngcf_dropout_widths(gpu, dims, td):
    """'philox' mess 0.3 + node 0.2 at widths that are not multiples of 4 (the scalar mix kernels, mask chunks o >> 2 that
    straddle rows) and at 256: the forward and the backward must use the same mask"""
    ops = gpu
    rng = np.random.default_rng(100 + sum(dims) + td)
    U, I = 1500, 1200
    adj = random_graph(rng, U, I, 20000)
    graph, rg = ops.LgcnGraph(*adj, "cuda"), RefGraph(*adj, "cuda")
    E0, W = _tables(ops, rng, U, I, dims)
    B = 3000
    planes = planes_uniform(rng, U, I, 2 * B)

    def make(opt, lr):
        return DropGpu(graph, rg, U, I, E0, W, planes, len(dims) - 1, opt, lr, (1e-3, 1e-3), dims, td, seed=5 + td, mess=0.3,
                       node=0.2)
    report(f"ngcf dropout widths {dims} td={td}", _sgd_then_adam(make, B, f"{dims} td={td}", 11))


# ---------------------------------------------------------------- GPU: launches
@pytest.mark.gpu
@pytest.mark.parametrize("td", [0, 1])
def test_ngcf_dropout_launches(gpu, td):
    """one 3-step 'philox' launch (first_step 2, forward0 5, short last batch) against three single launches at forward
    counters 5, 6, 7, each checked; a loss-only call on an Adam workspace leaves E0, W and the moments alone and needs no
    mirror index"""
    ops = gpu
    dims = [32, 32, 16]
    rng = np.random.default_rng(40 + td)
    U, I = 1500, 1200
    adj = random_graph(rng, U, I, 20000)
    assert np.diff(adj[0]).max() > 256
    graph, rg = ops.LgcnGraph(*adj, "cuda"), RefGraph(*adj, "cuda")
    E0, W = _tables(ops, rng, U, I, dims)
    B = 2000
    T = 5 * B - 500
    planes = planes_uniform(rng, U, I, T)
    kw = dict(seed=909, mess=0.1, node=0.2)
    multi = DropGpu(graph, rg, U, I, E0, W, planes, 2, "sgd", 0.05, (1e-3, 1e-3), dims, td, forward0=5, **kw)
    single = DropGpu(graph, rg, U, I, E0, W, planes, 2, "sgd", 0.05, (1e-3, 1e-3), dims, td, **kw)
    recs = launch_vs_singles(multi, single, T, B, 3, first_step=2, step_of=lambda s: single.masks(5 + s - 2))
    assert recs[2]["nb"] == B - 500
    ad = DropGpu(graph, rg, U, I, E0, W, planes, 2, "adam", 0.001, (1e-3, 1e-3), dims, td, **kw)
    recs.append(checked_step(ad, 0, B, B, "adam step 0", ref_device="cuda", **ad.masks(8)))
    ad.graph = fresh = ops.LgcnGraph(*adj, "cuda")
    recs.append(checked_step(ad, B, B, B, "loss only", adam_step0=1, apply=False, ref_device="cuda", **ad.masks(9)))
    assert fresh.mirror is None
    report(f"ngcf dropout launches td={td}", recs)


# ---------------------------------------------------------------- GPU: the scoring forward
@pytest.mark.gpu
@pytest.mark.parametrize("td", [0, 1])
@pytest.mark.parametrize("dims", [[64, 64, 64, 64], [256, 256]], ids=lambda d: "-".join(map(str, d)))
def test_ngcf_forward_philox(gpu, dims, td):
    """ngcf_forward_philox against the float64 forward with the same masks: message dropout alone (the forward rank() runs
    after fit) and with node dropout"""
    ops = gpu
    rng = np.random.default_rng(7 + len(dims) + td)
    U, I = 1500, 1200
    adj = random_graph(rng, U, I, 20000)
    graph, rg = ops.LgcnGraph(*adj, "cuda"), RefGraph(*adj, "cuda")
    E0, W = _tables(ops, rng, U, I, dims)
    ws = ops.NgcfWorkspace(U, I, dims, "sgd", "cuda")
    for mess, node in ((0.1, 0.0), (0.3, 0.2)):
        keep, edge = ops.ngcf_philox_masks(13, 4, U, I, dims, mess, node, len(adj[1]), "cuda")
        got = ops.ngcf_forward_philox(E0, W, ws, graph, tower_dtype=td, seed=13, forward=4, mess_dropout=mess, node_dropout=node)
        r, need = ngcf_forward_check(ops, graph, rg, U, I, E0, W, dims, td, keep, mess, edge if node > 0 else None, node, got=got)
        print(f"forward philox {dims} td={td} mess={mess} node={node}: worst error/bound {r:.3g}, kappa needed {need:.3g}")
        assert r <= 1, (mess, node, r)


# ---------------------------------------------------------------- GPU: the mirror index
@pytest.mark.gpu
def test_edge_mirror_amazon_book(gpu):
    """graph.edge_mirror() at the Amazon-Book adjacency: the slot order of (col, row), an involution, and the reference's
    A_drop^T reads A_drop at the mirror slot; an adjacency that is not structurally symmetric raises ValueError"""
    ops = gpu
    U, I, graph, rg, planes, g = amazon_book(1024, 1)
    rp, col = rg.row_ptr.numpy(), rg.col.numpy()
    nnz = len(col)
    rows = np.repeat(np.arange(rg.n), np.diff(rp))
    mirror = graph.edge_mirror()[:nnz].cpu().numpy()
    assert np.array_equal(mirror, np.lexsort((rows, col)))
    assert np.array_equal(mirror[mirror], np.arange(nnz))
    edge = (np.random.default_rng(1).random(nnz) >= 0.3).astype(np.uint8)
    d = rg.dropped_by(edge, 0.3)
    assert np.array_equal(d.T.val.numpy(), d.val.numpy()[mirror]) and np.array_equal(d.T.col.numpy(), col)
    # row 0 loses its last stored entry: its mirror slot has no partner
    r0 = int(rp[1]) - 1
    keep = np.arange(nnz) != r0
    asym = ops.LgcnGraph(np.concatenate([[0], np.cumsum(np.bincount(rows[keep], minlength=rg.n))]), col[keep],
                         rg.val.numpy()[keep], "cuda")
    with pytest.raises(ValueError, match="structurally symmetric"):
        asym.edge_mirror()


# ---------------------------------------------------------------- CPU: the bound sees dropout defects
class DropStandIn(StandIn):
    """the fp32 stand-in with dropout; defect msg_mask_stale: step s runs on the masks of the step before"""
    prev = None

    def stand_in_ref(self, idx, **step):
        use = dict(step, keep=self.prev["keep"]) if "msg_mask_stale" in self.defects and self.prev is not None else step
        self.prev = step
        return self.reference(self.t, idx, self.kappa, torch.float32, self.defects, **use)


def _cpu_drop(opt="sgd", td=0, defects=(), mess=0.2, node=0.3, seed=11):
    st, rg, B = _cpu_case("ngcf", seed=seed, opt=opt, td=td, reg=(0.0, 0.0) if opt == "adam" else (1e-3, 1e-3),
                          defects=defects, cls=DropStandIn)
    assert np.diff(rg.row_ptr.numpy()).max() > 256
    rng = np.random.default_rng(seed + 1)
    n = st.U + st.I

    def masks(s):
        return dict(keep=torch.from_numpy((rng.random(n * sum(st.dims[1:])) >= mess).astype(np.uint8)), p=mess,
                    edge=torch.from_numpy((rng.random(rg.col.numel()) >= node).astype(np.uint8)), node_p=node, forward=s)
    return st, B, masks


@pytest.mark.parametrize("opt,td", [("sgd", 0), ("adam", 0), ("sgd", 1), ("adam", 1)])
def test_harness_passes_with_fp32_stand_in_dropout(opt, td):
    st, B, masks = _cpu_drop(opt, td)
    for s in range(2):
        r = checked_step(st, s * B, B, B, f"stand-in dropout {opt} td={td} {s}", adam_step0=s, **masks(s))
        assert r["ok"], summary(r)


DROP_DEFECTS = {
    # defect: the tensors at least one of which must exceed the bound
    "node_bwd_untransposed": {"E0"},
    "node_mask_per_layer": {"E0", "W1[1]", "W2[1]", "b1[1]", "b2[1]"},
    "node_unscaled": {"E0", "W1[0]", "W2[0]"},
    "msg_bwd_unmasked": {"E0", "W1[0]", "W2[0]", "W1[1]", "W2[1]", "b1[1]", "b2[1]"},
    "msg_mask_stale": {"E0", "W1[0]", "W2[0]", "W1[1]", "W2[1]", "b1[1]", "b2[1]"},
}


@pytest.mark.parametrize("defect", sorted(DROP_DEFECTS))
def test_harness_flags_dropout_defect(defect):
    """each defect fails the bound on the named tensors at the second of two steps; the same run without it passes"""
    for defects in ((defect,), ()):
        st, B, masks = _cpu_drop(defects=defects)
        recs = [checked_step(st, s * B, B, B, f"{defect} {s}" if defects else f"no defect {s}", **masks(s)) for s in range(2)]
        if not defects:
            assert all(r["ok"] for r in recs), [summary(r) for r in recs]
            continue
        r = recs[1]
        bad = {k for k, v in r["tensors"].items() if v["ratio"] > 1 or v["unflagged"] > 0}
        print(f"{defect}: worst error/bound {r['ratio']:.3g} at {r['worst_at']}; over the bound: {sorted(bad)}")
        assert not r["ok"], summary(r)
        assert bad & DROP_DEFECTS[defect], (defect, bad)
