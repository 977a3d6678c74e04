"""wgmma (bf16 operands, fp32 register accumulators) GEMM of the NeuMF tower vs a float64 product of the bf16-rounded
operands, and the bf16-tower training step vs the fp32 tower (BASELINE config 3 tolerance)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from daisyrec_b200 import ops as o
    o.require_cuda()
    return o


def bf(x):
    return x.to(torch.bfloat16).to(torch.float64)


@pytest.mark.parametrize("M,N,K", [(1000, 64, 128), (4096, 32, 64), (300, 24, 48), (129, 128, 32), (77, 16, 200), (2048, 256, 96)])
def test_umma_forward_nt_bias_relu(ops, M, N, K):
    g = torch.Generator(device="cuda"); g.manual_seed(M + N + K)
    A = torch.randn(M, K, device="cuda", generator=g)
    W = torch.randn(N, K, device="cuda", generator=g) * 0.2
    b = torch.randn(N, device="cuda", generator=g)
    want = torch.relu(bf(A) @ bf(W).T + b.double()).float()
    for dtype in (0, 1):
        C = torch.full((M, N), -7.0, device="cuda")
        ops.gemm_test(0, dtype, A, W, C, M, N, K, bias=b)
        torch.cuda.synchronize()
        ref = want if dtype == 1 else torch.relu(A.double() @ W.double().T + b.double()).float()
        tol = 1e-4 * max(1.0, float(ref.abs().max()))
        assert float((C - ref).abs().max()) <= tol, (dtype, float((C - ref).abs().max()))


@pytest.mark.parametrize("M,N,K", [(777, 128, 64), (1024, 64, 32), (500, 96, 48)])
def test_umma_input_gradient_nn_mask(ops, M, N, K):
    g = torch.Generator(device="cuda"); g.manual_seed(M * 3 + N)
    dZ = torch.randn(M, K, device="cuda", generator=g)
    W = torch.randn(K, N, device="cuda", generator=g) * 0.3          # [out, in] row-major
    ref_act = torch.randn(M, N, device="cuda", generator=g)
    want = ((bf(dZ) @ bf(W)) * (ref_act > 0)).float()
    C = torch.zeros(M, N, device="cuda")
    ops.gemm_test(1, 1, dZ, W, C, M, N, K, ref=ref_act)
    assert float((C - want).abs().max()) <= 1e-4 * max(1.0, float(want.abs().max()))
    C2 = torch.zeros(M, N, device="cuda")
    ops.gemm_test(2, 1, dZ, W, C2, M, N, K)
    assert float((C2 - (bf(dZ) @ bf(W)).float()).abs().max()) <= 1e-4 * max(1.0, float(want.abs().max()))


@pytest.mark.parametrize("Mo,Ni,R", [(64, 128, 5000), (32, 64, 70000), (24, 48, 999), (128, 256, 4096)])
def test_umma_weight_gradient_tn_splitk(ops, Mo, Ni, R):
    g = torch.Generator(device="cuda"); g.manual_seed(Mo + Ni + R)
    dZ = torch.randn(R, Mo, device="cuda", generator=g) * 0.1
    X = torch.randn(R, Ni, device="cuda", generator=g)
    want = (bf(dZ).T @ bf(X)).float()
    C = torch.zeros(Mo, Ni, device="cuda")
    ops.gemm_test(3, 1, dZ, X, C, Mo, Ni, R)
    assert float((C - want).abs().max()) <= 2e-4 * max(1.0, float(want.abs().max()))


@pytest.mark.parametrize("Mi,No,R", [(128, 64, 5000), (64, 32, 70000), (48, 24, 999), (256, 128, 4096)])
def test_umma_weight_gradient_transposed_accumulate(ops, Mi, No, R):
    """variant 4 (what the tower uses): gW[out, in] += (X^T dZ)^T with the wide dimension on the MMA rows."""
    g = torch.Generator(device="cuda"); g.manual_seed(Mi + No + R)
    X = torch.randn(R, Mi, device="cuda", generator=g)
    dZ = torch.randn(R, No, device="cuda", generator=g) * 0.1
    want = (bf(dZ).T @ bf(X)).float()                                   # [out, in]
    for dtype in (0, 1):
        C = torch.zeros(No, Mi, device="cuda")
        ops.gemm_test(4, dtype, X, dZ, C, Mi, No, R)
        ref = want if dtype == 1 else (dZ.double().T @ X.double()).float()
        assert float((C - ref).abs().max()) <= 2e-4 * max(1.0, float(ref.abs().max())), dtype


def test_neumf_bf16_tower_step_close_to_fp32(ops):
    """One NeuMF step with the wgmma bf16 tower vs the fp32 tower: loss within 2e-3 relative, tables within bf16 noise."""
    rng = np.random.default_rng(0)
    U, I, F, L, B = 500, 400, 32, 2, 4096
    D = F * 2 ** (L - 1)
    tabs_h = [(rng.standard_normal(s) * 0.2).astype(np.float32) for s in ((U, F), (I, F), (U, D), (I, D))]
    W_h = (rng.standard_normal(ops.neumf_param_count(F, L)) * 0.15).astype(np.float32)
    b = [torch.from_numpy(rng.integers(m, size=B).astype(np.int32)).cuda() for m in (U, I, I)]
    hp = ops.hyper(0.01, 0.001, 0.001, "sgd")
    res = []
    for dtype in (0, 1):
        tabs = [torch.from_numpy(t).cuda() for t in tabs_h]
        W = torch.from_numpy(W_h).cuda()
        ws = ops.NeumfWorkspace(U, I, F, L, "sgd", 2 * B, "cuda")
        loss = ops.neumf_bpr_train_steps(tabs, W, ws, *b, B, 0, 1, hp, tower_dtype=dtype).item()
        res.append((loss, [t.cpu().numpy() for t in tabs], W.cpu().numpy()))
    (l0, t0, w0), (l1, t1, w1) = res
    assert abs(l1 - l0) <= 2e-3 * abs(l0), (l0, l1)
    # compare the UPDATES in norm: bf16 operands perturb every product by ~2^-8 and flip the ReLU gate of the few
    # pre-activations that sit at zero, so single elements can move by O(10 %) while the update as a whole agrees
    for init, a, c in zip(tabs_h + [W_h], t0 + [w0], t1 + [w1]):
        d_fp32, d_bf16 = (a - init).astype(np.float64), (c - init).astype(np.float64)
        rel = np.linalg.norm(d_bf16 - d_fp32) / max(np.linalg.norm(d_fp32), 1e-30)
        cos = float((d_bf16 * d_fp32).sum() / max(np.linalg.norm(d_bf16) * np.linalg.norm(d_fp32), 1e-30))
        assert rel <= 0.15 and cos >= 0.99, (rel, cos)


@pytest.mark.parametrize("B,reg", [(64, 0.0), (4096, 0.001), (5000, 0.002), (130, 0.001)])
def test_neumf_fused_tower_matches_layerwise_bf16(ops, B, reg):
    """tower_dtype 2 (the whole tower step of a 64-triple tile fused in one CTA: bf16 operand images in shared memory, every
    accumulator in registers, transposed operands read through swapped-stride descriptors) against tower_dtype 1 (the same bf16
    products as separate GEMM launches).  Both round the same values to bf16 at the same points, so they agree to fp32
    accumulation-order noise: a wrong descriptor, fragment column or image offset shows up as an O(1) error in exactly one of
    {loss (forward), embedding tables (dZ W products), tower block (A^T dZ products, bias / predict sums)}."""
    rng = np.random.default_rng(B)
    U, I, F, L = 700, 500, 32, 2
    D = F * 2 ** (L - 1)
    tabs_h = [(rng.standard_normal(s) * 0.2).astype(np.float32) for s in ((U, F), (I, F), (U, D), (I, D))]
    W_h = (rng.standard_normal(ops.neumf_param_count(F, L)) * 0.15).astype(np.float32)
    b = [torch.from_numpy(rng.integers(m, size=B).astype(np.int32)).cuda() for m in (U, I, I)]
    hp = ops.hyper(0.01, reg, reg, "sgd")
    res = []
    for dtype in (1, 2):
        tabs = [torch.from_numpy(t).cuda() for t in tabs_h]
        W = torch.from_numpy(W_h).cuda()
        ws = ops.NeumfWorkspace(U, I, F, L, "sgd", 2 * B, "cuda")
        l0 = ops.neumf_bpr_train_steps(tabs, W, ws, *b, B, 0, 1, hp, tower_dtype=dtype, apply=False).item()
        assert all(np.array_equal(t.cpu().numpy(), h) for t, h in zip(tabs, tabs_h))      # loss-only call changes nothing
        loss = ops.neumf_bpr_train_steps(tabs, W, ws, *b, B, 0, 1, hp, tower_dtype=dtype).item()
        assert l0 == loss or abs(l0 - loss) <= 1e-6 * abs(loss)
        res.append((loss, [t.cpu().numpy() for t in tabs], W.cpu().numpy()))
    (l1, t1, w1), (l2, t2, w2) = res
    assert abs(l2 - l1) <= 2e-5 * abs(l1), ("forward", l1, l2)
    names = ["UG", "IG", "UM", "IM"]
    for n, init, a, c in zip(names, tabs_h, t1, t2):
        upd = np.abs(a - init).max()
        assert np.abs(c - a).max() <= 2e-4 * max(upd, 1e-12) + 1e-9, (n, float(np.abs(c - a).max()), float(upd))
    n1, n0, n2 = 2 * F, 4 * F, F
    blocks = {"W1": (0, n1 * n0), "b1": (n1 * n0, n1 * n0 + n1), "W2": (n1 * n0 + n1, n1 * n0 + n1 + n2 * n1),
              "b2": (n1 * n0 + n1 + n2 * n1, n1 * n0 + n1 + n2 * n1 + n2), "wp": (n1 * n0 + n1 + n2 * n1 + n2, len(W_h))}
    for n, (lo, hi) in blocks.items():
        upd = np.abs(w1[lo:hi] - W_h[lo:hi]).max()
        assert np.abs(w2[lo:hi] - w1[lo:hi]).max() <= 5e-4 * max(upd, 1e-12) + 1e-9, (n, float(np.abs(w2[lo:hi] - w1[lo:hi]).max()), float(upd))


def test_neumf_fused_tower_multi_step_training(ops):
    """Several chained Adam steps over many tiles per CTA (register weight-gradient accumulators carried across tiles, flushed once)."""
    rng = np.random.default_rng(9)
    U, I, F, L, B, K = 3000, 2000, 32, 2, 20000, 3
    D = F * 2 ** (L - 1)
    tabs_h = [(rng.standard_normal(s) * 0.1).astype(np.float32) for s in ((U, F), (I, F), (U, D), (I, D))]
    W_h = (rng.standard_normal(ops.neumf_param_count(F, L)) * 0.1).astype(np.float32)
    b = [torch.from_numpy(rng.integers(m, size=B * K).astype(np.int32)).cuda() for m in (U, I, I)]
    hp = ops.hyper(0.001, 0.001, 0.001, "adam")
    out = []
    for dtype in (1, 2):
        tabs = [torch.from_numpy(t).cuda() for t in tabs_h]
        W = torch.from_numpy(W_h).cuda()
        ws = ops.NeumfWorkspace(U, I, F, L, "adam", 2 * B, "cuda")
        losses = ops.neumf_bpr_train_steps(tabs, W, ws, *b, B, 0, K, hp, tower_dtype=dtype).cpu().numpy()
        out.append((losses, W.cpu().numpy(), tabs[2].cpu().numpy()))
    (la, wa, ta), (lb, wb, tb) = out
    assert np.all(np.abs(la - lb) <= 1e-4 * np.abs(la)), (la, lb)
    # Adam normalises every gradient to ~lr: compare the direction of the accumulated update
    for a, c, init in ((wa, wb, W_h), (ta, tb, tabs_h[2])):
        da, dc = (a - init).astype(np.float64).ravel(), (c - init).astype(np.float64).ravel()
        cos = float(da @ dc / max(np.linalg.norm(da) * np.linalg.norm(dc), 1e-30))
        assert cos >= 0.995, cos
