"""Tensor-level bindings of the C ABI (include/daisyrec_b200.h).

torch is plumbing here: device memory (``tensor.data_ptr()``) and the current CUDA stream.
Every function forwards to libdaisyrec_b200.so; nothing is computed by torch ops.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib as L


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return C.c_void_p(t.data_ptr())


def _dev(t, dtype, name):
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == dtype and t.is_contiguous()):
        raise TypeError(f"{name}: expected a contiguous CUDA tensor of dtype {dtype}")
    return t


def _train_steps(fn, n_steps, device, check, *args, out=None):
    """Calls a step entry point with ``args`` followed by its trailing (d_step_loss, sync_and_check, nan_step, stream)
    arguments -> float64 device losses [n_steps] (in ``out`` when given)."""
    losses = out if out is not None else torch.empty(max(n_steps, 1), dtype=torch.float64, device=device)
    nan_step = C.c_int64(-1)
    L.check(fn(*args, _ptr(losses), 1 if check else 0, C.byref(nan_step), _stream()))
    return losses[:n_steps]


def require_cuda():
    if not torch.cuda.is_available():
        raise RuntimeError("daisyrec_b200 needs a CUDA device (sm_90a); there is no CPU fallback")


def hyper(lr, reg_1, reg_2, opt="sgd", beta1=0.9, beta2=0.999, eps=1e-8, loss="BPR"):
    return L.Hyper(lr, reg_1, reg_2, L.OPT_KIND[opt], beta1, beta2, eps, L.LOSS_KIND[loss.upper()])


def device_query():
    sm, ma, mi, l2 = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int64()
    L.check(L.lib().drb_device_query(C.byref(sm), C.byref(ma), C.byref(mi), C.byref(l2)))
    return dict(sm_count=sm.value, cc=(ma.value, mi.value), l2_bytes=l2.value)


def mf_step_variant(factors, table_rows=0):
    """-> (lean, lanes_per_row, chunks_per_lane) of the BPR + SGD / Adam step kernel for this factor count and table size
    (user_num + item_num; 0 = the L2 regime).  Runs the one-off on-device selection if it has not run yet."""
    w, n = C.c_int32(0), C.c_int32(0)
    lean = L.lib().drb_mf_step_variant(int(factors), int(table_rows), C.byref(w), C.byref(n))
    return bool(lean), int(w.value), int(n.value)


def mf_step_selfcheck_ms(factors, table_rows=0):
    """-> (ms_general, ms_lean, tile_cap) of the on-device selection for this factor count and table size."""
    a, b, t = C.c_float(0), C.c_float(0), C.c_int32(0)
    L.lib().drb_mf_step_selfcheck_ms(int(factors), int(table_rows), C.byref(a), C.byref(b), C.byref(t))
    return float(a.value), float(b.value), int(t.value)


def check_index_range(ids, bounds, what):
    """IndexError (what nn.Embedding raises in the reference) when a column of the device index array ``ids`` [n, len(bounds)]
    holds an id outside [0, bounds[c]).  One kernel + one 64-byte read-back."""
    if not (isinstance(ids, torch.Tensor) and ids.is_cuda and ids.is_contiguous() and ids.dtype in (torch.int32, torch.int64)):
        raise TypeError("check_index_range: expected a contiguous CUDA int32 / int64 tensor")
    ncols = len(bounds)
    n = ids.numel() // ncols
    hi = (C.c_int64 * 4)(*([int(b) for b in bounds] + [0] * (4 - ncols)))
    bad = (C.c_int64 * 4)()
    L.check(L.lib().drb_index_range_check(_ptr(ids), ids.element_size(), n, ncols, hi, bad, _stream()))
    for c in range(ncols):
        if bad[c]:
            raise IndexError(f"index out of range in self: {bad[c]} {what[c]} id(s) outside [0, {int(bounds[c])})")


# ------------------------------------------------------------------ sampler
def mt19937_seed(seed):
    st = np.zeros(625, np.uint32)
    L.check(L.lib().drb_mt19937_seed(st.ctypes.data, C.c_uint32(seed & 0xFFFFFFFF)))
    return st


def mt19937_from_numpy(rs=None):
    s = (np.random if rs is None else rs).get_state()
    st = np.zeros(625, np.uint32)
    st[:624] = s[1]
    st[624] = s[2]
    return st


def mt19937_to_numpy(st, rs=None):
    tgt = np.random if rs is None else rs
    old = tgt.get_state()
    tgt.set_state(("MT19937", st[:624].copy(), int(st[624]), old[3], old[4]))


def sampler_draw_mt19937(state, row_ptr, user_num, item_num, num_ng):
    """Host: the reference's per-user bounded draws (advances ``state`` in place)."""
    row_ptr = np.ascontiguousarray(row_ptr, np.int64)
    draws = np.empty((user_num, num_ng), np.int32)
    bad = C.c_int32(-1)
    rc = L.lib().drb_sampler_draw_mt19937(state.ctypes.data, row_ptr.ctypes.data, user_num, item_num, num_ng,
                                          draws.ctypes.data, C.byref(bad))
    L.check(rc)
    return draws


def sampler_draw_philox(seed, offset, d_row_ptr, user_num, item_num, num_ng):
    _dev(d_row_ptr, torch.int64, "row_ptr")
    draws = torch.empty((user_num, num_ng), dtype=torch.int32, device=d_row_ptr.device)
    bad = torch.empty(1, dtype=torch.int32, device=d_row_ptr.device)
    L.check(L.lib().drb_sampler_draw_philox(C.c_uint64(seed), C.c_uint64(offset), _ptr(d_row_ptr), user_num, item_num,
                                            num_ng, _ptr(draws), _ptr(bad), _stream()))
    return draws, bad


def sampler_kth_complement(d_row_ptr, d_col, d_draws, item_num):
    _dev(d_row_ptr, torch.int64, "row_ptr"); _dev(d_col, torch.int32, "col"); _dev(d_draws, torch.int32, "draws")
    U, G = d_draws.shape
    js = torch.empty_like(d_draws)
    L.check(L.lib().drb_sampler_kth_complement(_ptr(d_row_ptr), _ptr(d_col), _ptr(d_draws), U, item_num, G, _ptr(js),
                                               _stream()))
    return js


def sampler_explode(d_coo_u, d_coo_i, d_js):
    _dev(d_coo_u, torch.int32, "coo_u"); _dev(d_coo_i, torch.int32, "coo_i"); _dev(d_js, torch.int32, "js")
    nnz, G = d_coo_u.numel(), d_js.shape[1]
    tr = torch.empty((nnz * G, 3), dtype=torch.int32, device=d_js.device)
    L.check(L.lib().drb_sampler_explode(_ptr(d_coo_u), _ptr(d_coo_i), nnz, _ptr(d_js), G, _ptr(tr), _stream()))
    return tr


def sample_triples_host(state, row_ptr, col, coo_u, coo_i, user_num, item_num, num_ng):
    """All-host-buffer convenience call (H2D/D2H inside the library)."""
    row_ptr = np.ascontiguousarray(row_ptr, np.int64)
    col = np.ascontiguousarray(col, np.int32)
    coo_u = np.ascontiguousarray(coo_u, np.int32)
    coo_i = np.ascontiguousarray(coo_i, np.int32)
    js = np.empty((user_num, num_ng), np.int32)
    tr = np.empty((len(coo_u) * num_ng, 3), np.int32)
    bad = C.c_int32(-1)
    rc = L.lib().drb_sample_triples_host(state.ctypes.data, row_ptr.ctypes.data, col.ctypes.data, coo_u.ctypes.data,
                                         coo_i.ctypes.data, len(coo_u), user_num, item_num, num_ng, js.ctypes.data,
                                         tr.ctypes.data, C.byref(bad))
    L.check(rc)
    return js, tr


def bounded_draws_mt19937(state, n, offsets):
    """Host: row m draws offsets[m+1]-offsets[m] values from [0, n[m]) off numpy's MT19937 stream."""
    n = np.ascontiguousarray(n, np.int64)
    offsets = np.ascontiguousarray(offsets, np.int64)
    draws = np.empty(int(offsets[-1]), np.int32)
    bad = C.c_int64(-1)
    rc = L.lib().drb_bounded_draws_mt19937(state.ctypes.data, n.ctypes.data, offsets.ctypes.data, len(n),
                                           draws.ctypes.data, C.byref(bad))
    L.check(rc)
    return draws


def kth_complement_var(d_row_ptr, d_col, d_offsets, d_draws):
    _dev(d_row_ptr, torch.int64, "row_ptr"); _dev(d_col, torch.int32, "col")
    _dev(d_offsets, torch.int64, "offsets"); _dev(d_draws, torch.int32, "draws")
    out = torch.empty_like(d_draws)
    L.check(L.lib().drb_kth_complement_var(_ptr(d_row_ptr), _ptr(d_col), _ptr(d_offsets), _ptr(d_draws),
                                           d_row_ptr.numel() - 1, _ptr(out), _stream()))
    return out


def sampler_draw_mt19937_mixed(state, row_ptr, user_num, item_num, uniform_num, other_num):
    """Host: numpy-stream replay of the popularity-mixed branch (sampler.py:71-80) -> (ranks i32, doubles f64)."""
    row_ptr = np.ascontiguousarray(row_ptr, np.int64)
    draws = np.empty((user_num, uniform_num), np.int32)
    u01 = np.empty((user_num, other_num), np.float64)
    bad = C.c_int32(-1)
    rc = L.lib().drb_sampler_draw_mt19937_mixed(state.ctypes.data, row_ptr.ctypes.data, user_num, item_num, uniform_num,
                                                other_num, draws.ctypes.data, u01.ctypes.data, C.byref(bad))
    L.check(rc)
    return draws, u01


def sampler_assemble_mixed(d_row_ptr, d_col, d_draws, d_cdf, d_u01, item_num):
    _dev(d_row_ptr, torch.int64, "row_ptr"); _dev(d_col, torch.int32, "col")
    _dev(d_draws, torch.int32, "draws"); _dev(d_cdf, torch.float64, "cdf"); _dev(d_u01, torch.float64, "u01")
    U, un, on = d_row_ptr.numel() - 1, d_draws.shape[1], d_u01.shape[1]
    js = torch.empty((U, un + on), dtype=torch.int32, device=d_row_ptr.device)
    L.check(L.lib().drb_sampler_assemble_mixed(_ptr(d_row_ptr), _ptr(d_col), _ptr(d_draws), _ptr(d_cdf), _ptr(d_u01), U,
                                               item_num, un, on, _ptr(js), _stream()))
    return js


def sampler_explode_pointwise(d_coo_u, d_coo_i, d_label, d_js):
    _dev(d_coo_u, torch.int32, "coo_u"); _dev(d_coo_i, torch.int32, "coo_i")
    _dev(d_label, torch.int32, "label"); _dev(d_js, torch.int32, "js")
    nnz, G = d_coo_u.numel(), d_js.shape[1]
    rows = torch.empty((nnz * (1 + G), 3), dtype=torch.int32, device=d_coo_u.device)
    L.check(L.lib().drb_sampler_explode_pointwise(_ptr(d_coo_u), _ptr(d_coo_i), _ptr(d_label), nnz, _ptr(d_js), G,
                                                  _ptr(rows), _stream()))
    return rows


# ------------------------------------------------------------------ CSR / adjacency builders
def skipgram_group(d_coo_u, user_num, window):
    """Device: (seq_ptr int64 [U+1], ctx_ptr int64 [U+1], order int32 [nnz]) -- the train rows grouped by user in row order."""
    _dev(d_coo_u, torch.int32, "coo_u")
    n, dev = d_coo_u.numel(), d_coo_u.device
    ws = torch.empty(max(1, L.lib().drb_skipgram_workspace_bytes(user_num, n)), dtype=torch.uint8, device=dev)
    seq_ptr = torch.empty(user_num + 1, dtype=torch.int64, device=dev)
    ctx_ptr = torch.empty(user_num + 1, dtype=torch.int64, device=dev)
    order = torch.empty(max(1, n), dtype=torch.int32, device=dev)
    L.check(L.lib().drb_skipgram_group(_ptr(d_coo_u), n, user_num, window, _ptr(ws), _ptr(seq_ptr), _ptr(ctx_ptr),
                                       _ptr(order), _stream()))
    return seq_ptr, ctx_ptr, order[:n]


def skipgram_draws_mt19937(state, n, seq_len, window, total):
    """Host: the ``total`` negative ranks of the skip-gram sampler off numpy's MT19937 stream (advances ``state``)."""
    n = np.ascontiguousarray(n, np.int64)
    seq_len = np.ascontiguousarray(seq_len, np.int64)
    draws = np.empty(max(1, total), np.int32)
    bad = C.c_int32(-1)
    L.check(L.lib().drb_skipgram_draws_mt19937(state.ctypes.data, n.ctypes.data, seq_len.ctypes.data, len(n), window,
                                               draws.ctypes.data, C.byref(bad)))
    return draws[:total]


def skipgram_emit(d_coo_u, d_coo_i, d_order, window, d_seq_ptr, d_ctx_ptr, d_row_ptr, d_col, d_draws, total):
    """Device: int32 [2 * total, 3] skip-gram rows."""
    for t, nm in ((d_coo_u, "coo_u"), (d_coo_i, "coo_i"), (d_order, "order"), (d_col, "col"), (d_draws, "draws")):
        _dev(t, torch.int32, nm)
    for t, nm in ((d_seq_ptr, "seq_ptr"), (d_ctx_ptr, "ctx_ptr"), (d_row_ptr, "row_ptr")):
        _dev(t, torch.int64, nm)
    rows = torch.empty((2 * total, 3), dtype=torch.int32, device=d_coo_u.device)
    L.check(L.lib().drb_skipgram_emit(_ptr(d_coo_u), _ptr(d_coo_i), _ptr(d_order), d_order.numel(), window, _ptr(d_seq_ptr),
                                      _ptr(d_ctx_ptr), _ptr(d_row_ptr), _ptr(d_col), _ptr(d_draws), _ptr(rows), _stream()))
    return rows


def csr_build(d_row, d_col, n_rows, n_cols):
    """COO int32 pairs on the device -> (row_ptr int64[n_rows+1], col int32[nnz_unique]) sorted + duplicate-free."""
    _dev(d_row, torch.int32, "row"); _dev(d_col, torch.int32, "col")
    nnz = d_row.numel()
    ws = torch.empty(L.lib().drb_csr_workspace_bytes(n_rows, nnz), dtype=torch.uint8, device=d_row.device)
    row_ptr = torch.empty(n_rows + 1, dtype=torch.int64, device=d_row.device)
    col = torch.empty(max(nnz, 1), dtype=torch.int32, device=d_row.device)
    kept = C.c_int64(0)
    L.check(L.lib().drb_csr_build(_ptr(d_row), _ptr(d_col), nnz, n_rows, n_cols, _ptr(ws), _ptr(row_ptr), _ptr(col),
                                  C.byref(kept), _stream()))
    return row_ptr, col[:kept.value]


def lgcn_build_adj(d_coo_u, d_coo_i, user_num, item_num):
    """Train COO on the device -> A_hat CSR (row_ptr i64, col i32, val f32) of get_norm_adj_mat, built on the device."""
    ui_ptr, ui_col = csr_build(d_coo_u, d_coo_i, user_num, item_num)
    iu_ptr, iu_col = csr_build(d_coo_i, d_coo_u, item_num, user_num)
    nnz = ui_col.numel()
    assert iu_col.numel() == nnz
    dev = d_coo_u.device
    adj_ptr = torch.empty(user_num + item_num + 1, dtype=torch.int64, device=dev)
    adj_col = torch.empty(max(2 * nnz, 1), dtype=torch.int32, device=dev)
    adj_val = torch.empty(max(2 * nnz, 1), dtype=torch.float32, device=dev)
    L.check(L.lib().drb_lgcn_build_adj(_ptr(ui_ptr), _ptr(ui_col), _ptr(iu_ptr), _ptr(iu_col), user_num, item_num, nnz,
                                       _ptr(adj_ptr), _ptr(adj_col), _ptr(adj_val), _stream()))
    return adj_ptr, adj_col[:2 * nnz], adj_val[:2 * nnz]


# ------------------------------------------------------------------ evaluation KPIs
def rank_metrics(d_preds, d_gt_ptr, d_gt_idx, ks, item_num, d_item_pop=None):
    """calc_ranking_results' numbers for rank()'s device output: -> float64 CUDA tensor [len(ks), 8] (L.KPI_NAMES)."""
    _dev(d_preds, torch.float32, "preds"); _dev(d_gt_ptr, torch.int64, "gt_ptr"); _dev(d_gt_idx, torch.int32, "gt_idx")
    if d_item_pop is not None:
        _dev(d_item_pop, torch.float64, "item_pop")
    ks = np.ascontiguousarray(ks, np.int32)
    n, ld = d_preds.shape
    ws = torch.empty(L.lib().drb_rank_metrics_workspace_bytes(item_num, len(ks)), dtype=torch.uint8, device=d_preds.device)
    out = torch.empty((len(ks), len(L.KPI_NAMES)), dtype=torch.float64, device=d_preds.device)
    L.check(L.lib().drb_rank_metrics(_ptr(d_preds), n, ld, _ptr(d_gt_ptr), _ptr(d_gt_idx), ks.ctypes.data, len(ks),
                                     item_num, None if d_item_pop is None else _ptr(d_item_pop), _ptr(ws), _ptr(out),
                                     _stream()))
    return out


def rank_metrics_host(preds, gt_ptr, gt_idx, ks, item_num, item_pop=None):
    """Same through host buffers (H2D/D2H inside the library) -> float64 numpy [len(ks), 8]."""
    preds = np.ascontiguousarray(preds, np.float32)
    gt_ptr = np.ascontiguousarray(gt_ptr, np.int64)
    gt_idx = np.ascontiguousarray(gt_idx, np.int32)
    ks = np.ascontiguousarray(ks, np.int32)
    pop = None if item_pop is None else np.ascontiguousarray(item_pop, np.float64)
    out = np.empty((len(ks), len(L.KPI_NAMES)), np.float64)
    L.check(L.lib().drb_rank_metrics_host(preds.ctypes.data, preds.shape[0], preds.shape[1], gt_ptr.ctypes.data,
                                          gt_idx.ctypes.data, ks.ctypes.data, len(ks), item_num,
                                          None if pop is None else pop.ctypes.data, out.ctypes.data))
    return out


# ------------------------------------------------------------------ epoch permutation
def mt19937_stream(seed, n, device):
    out = torch.empty(max(n, 1), dtype=torch.int32, device=device)
    L.check(L.lib().drb_mt19937_stream(C.c_uint64(seed & 0xFFFFFFFFFFFFFFFF), n, _ptr(out), _stream()))
    return out[:n]


def mt19937_stream_variant(n):
    """'segmented' when drb_mt19937_stream runs the many-CTA jump-ahead kernel for n words (after its one-off device check),
    'one-cta' otherwise."""
    return "segmented" if L.lib().drb_mt19937_stream_variant(int(n)) else "one-cta"


def randperm_workspace(n, device):
    """(perm int64 [n], scratch) for randperm_torch(out=...): lets a caller keep them across epochs."""
    return (torch.empty(max(n, 1), dtype=torch.int64, device=device),
            torch.empty(L.lib().drb_randperm_workspace_bytes(n), dtype=torch.uint8, device=device))


def randperm_torch(seed, n, device, out=None):
    """torch.randperm(n, generator=G) for a CPU generator G with G.manual_seed(seed) -- computed on the device, bit-exact."""
    perm, ws = out if out is not None else randperm_workspace(n, device)
    L.check(L.lib().drb_randperm_torch(C.c_uint64(seed & 0xFFFFFFFFFFFFFFFF), n, _ptr(perm), _ptr(ws), _stream()))
    return perm[:n]


# ------------------------------------------------------------------ train feed
def gather_triples(d_triples, d_perm=None):
    _dev(d_triples, torch.int32, "triples")
    n = d_triples.shape[0] if d_perm is None else d_perm.numel()
    if d_perm is not None:
        _dev(d_perm, torch.int64, "perm")
    n4 = (n + 3) // 4 * 4                                   # 16-byte aligned planes for the TMA path
    soa = torch.empty((3, n4), dtype=torch.int32, device=d_triples.device)
    L.check(L.lib().drb_gather_triples(_ptr(d_triples), None if d_perm is None else _ptr(d_perm), n, _ptr(soa[0]),
                                       _ptr(soa[1]), _ptr(soa[2]), _stream()))
    return soa[0][:n], soa[1][:n], soa[2][:n]


# ------------------------------------------------------------------ training
class MFWorkspace:
    """Device scratch of the step kernel: gradient accumulators, row counters, optimiser state (Adam m, v; Adagrad /
    RMSprop one table)."""

    def __init__(self, user_num, item_num, factors, opt, device, deterministic=False):
        self.U, self.I, self.F = user_num, item_num, factors
        self.opt = L.OPT_KIND[opt]
        self.det = bool(deterministic)
        nbytes = (L.lib().drb_mf_workspace_bytes_det if self.det else L.lib().drb_mf_workspace_bytes)(user_num, item_num, factors,
                                                                                                     self.opt)
        self.buf = torch.empty(nbytes, dtype=torch.uint8, device=device)
        self.reset()

    def reset(self):
        if self.det:
            self.buf.zero_()               # the int64 images behind the regular layout as well
        else:
            L.check(L.lib().drb_mf_workspace_init(_ptr(self.buf), self.U, self.I, self.F, self.opt, _stream()))


def mf_bpr_train_steps(P, Q, ws, bu, bi, bj, batch, first_step, n_steps, hp, adam_step0=0, check=True, out=None):
    _dev(P, torch.float32, "P"); _dev(Q, torch.float32, "Q")
    for t, nm in ((bu, "bu"), (bi, "bi"), (bj, "bj")):
        _dev(t, torch.int32, nm)
    fn = L.lib().drb_mf_bpr_train_steps_det if getattr(ws, "det", False) else L.lib().drb_mf_bpr_train_steps
    return _train_steps(fn, n_steps, P.device, check, _ptr(P), _ptr(Q), _ptr(ws.buf), ws.U, ws.I, ws.F, _ptr(bu), _ptr(bi),
                        _ptr(bj), bu.numel(), batch, first_step, n_steps, C.byref(hp), adam_step0, out=out)


def mf_bpr_train_steps_fused_neg(P, Q, ws, bu, bi, d_row_ptr, d_col, seed, batch, first_step, n_steps, hp, adam_step0=0,
                                 neg_out=None, check=True):
    """Throughput mode: negatives are drawn inside the step kernel (fresh per triple and step) from the complement of the
    user's CSR row.  neg_out (optional int32 [n]) receives them."""
    _dev(P, torch.float32, "P"); _dev(Q, torch.float32, "Q"); _dev(bu, torch.int32, "bu"); _dev(bi, torch.int32, "bi")
    _dev(d_row_ptr, torch.int64, "row_ptr"); _dev(d_col, torch.int32, "col")
    return _train_steps(L.lib().drb_mf_bpr_train_steps_fused_neg, n_steps, P.device, check, _ptr(P), _ptr(Q), _ptr(ws.buf), ws.U,
                        ws.I, ws.F, _ptr(bu), _ptr(bi), _ptr(d_row_ptr), _ptr(d_col), C.c_uint64(seed),
                        None if neg_out is None else _ptr(neg_out), bu.numel(), batch, first_step, n_steps, C.byref(hp), adam_step0)


def mf_bpr_loss(P, Q, ws, bu, bi, bj, hp):
    _dev(P, torch.float32, "P"); _dev(Q, torch.float32, "Q")
    loss = torch.empty(1, dtype=torch.float64, device=P.device)
    L.check(L.lib().drb_mf_bpr_loss(_ptr(P), _ptr(Q), _ptr(ws.buf), ws.U, ws.I, ws.F, _ptr(bu), _ptr(bi), _ptr(bj),
                                    bu.numel(), C.byref(hp), _ptr(loss), _stream()))
    return loss


def stage_buffer(batch, device):
    stride = (batch + 3) // 4 * 4
    return torch.empty(3 * stride + 4, dtype=torch.int32, device=device)


def mf_bpr_train_step_host(P, Q, ws, h_bu, h_bi, h_bj, hp, stage, adam_step0=0):
    """One end-to-end step from HOST batch arrays (numpy int32 or CPU tensors, ideally pinned)."""
    def hp_(a):
        return a.data_ptr() if isinstance(a, torch.Tensor) else a.ctypes.data
    n = len(h_bu)
    loss = C.c_double(0.0)
    rc = L.lib().drb_mf_bpr_train_step_host(_ptr(P), _ptr(Q), _ptr(ws.buf), ws.U, ws.I, ws.F, hp_(h_bu), hp_(h_bi),
                                            hp_(h_bj), n, C.byref(hp), adam_step0, _ptr(stage), C.byref(loss), _stream())
    L.check(rc)
    return loss.value


def mf_bpr_train_steps_host(P, Q, ws, h_bu, h_bi, h_bj, batch, n_steps, hp, adam_step0=0):
    """Pipelined end-to-end steps from pinned HOST planes (CPU int32 tensors).  Returns float64 losses [n_steps]."""
    for t in (h_bu, h_bi, h_bj):
        if not (isinstance(t, torch.Tensor) and not t.is_cuda and t.dtype == torch.int32 and t.is_contiguous()):
            raise TypeError("host planes must be contiguous CPU int32 tensors (pin them for overlap)")
    n = h_bu.numel()
    stride = (batch + 3) // 4 * 4
    stage = torch.empty(2 * 3 * stride, dtype=torch.int32, device=P.device)
    d_loss = torch.empty(max(1, n_steps), dtype=torch.float64, device=P.device)
    h_loss = torch.empty(max(1, n_steps), dtype=torch.float64).pin_memory()
    nan_step = C.c_int64(-1)
    rc = L.lib().drb_mf_bpr_train_steps_host(_ptr(P), _ptr(Q), _ptr(ws.buf), ws.U, ws.I, ws.F, h_bu.data_ptr(),
                                             h_bi.data_ptr(), h_bj.data_ptr(), n, batch, n_steps, C.byref(hp), adam_step0,
                                             _ptr(stage), _ptr(d_loss), h_loss.data_ptr(), C.byref(nan_step), _stream())
    L.check(rc)
    return h_loss[:n_steps]


# ------------------------------------------------------------------ Item2Vec
class I2VWorkspace:
    """Step-kernel scratch of the one tied item table: gradient accumulator, row counters, Adam m and v."""

    def __init__(self, item_num, factors, opt, device):
        self.I, self.F = item_num, factors
        self.opt = L.OPT_KIND[opt]
        self.buf = torch.empty(L.lib().drb_i2v_workspace_bytes(item_num, factors, self.opt), dtype=torch.uint8, device=device)
        L.check(L.lib().drb_i2v_workspace_init(_ptr(self.buf), item_num, factors, self.opt, _stream()))


def i2v_train_steps(Q, ws, bt, bc, blabel, batch, first_step, n_steps, hp, adam_step0=0, apply=True, check=True):
    """Skip-gram steps on (target, context, label) planes; float64 device losses [n_steps].  apply=False: loss of one batch."""
    _dev(Q, torch.float32, "Q")
    for t, nm in ((bt, "target"), (bc, "context"), (blabel, "label")):
        _dev(t, torch.int32, nm)
    return _train_steps(L.lib().drb_i2v_train_steps, n_steps, Q.device, check, _ptr(Q), _ptr(ws.buf), ws.I, ws.F, _ptr(bt), _ptr(bc),
                        _ptr(blabel), bt.numel(), batch, first_step, n_steps, C.byref(hp), adam_step0, 1 if apply else 0)


def i2v_user_embedding(Q, d_row_ptr, d_col, P):
    """P[u] = sum of Q over the user's CSR row, for the users with a non-empty row (in place)."""
    _dev(Q, torch.float32, "Q"); _dev(P, torch.float32, "P")
    _dev(d_row_ptr, torch.int64, "row_ptr"); _dev(d_col, torch.int32, "col")
    L.check(L.lib().drb_i2v_user_embedding(_ptr(Q), Q.shape[1], _ptr(d_row_ptr), _ptr(d_col), P.shape[0], _ptr(P), _stream()))
    return P


# ------------------------------------------------------------------ FM
class FMWorkspace:
    """MF workspace + gradient accumulator / optimiser state of the packed bias vector."""

    def __init__(self, user_num, item_num, factors, opt, device):
        self.U, self.I, self.F = user_num, item_num, factors
        self.opt = L.OPT_KIND[opt]
        self.buf = torch.empty(L.lib().drb_fm_workspace_bytes(user_num, item_num, factors, self.opt), dtype=torch.uint8,
                               device=device)
        L.check(L.lib().drb_fm_workspace_init(_ptr(self.buf), user_num, item_num, factors, self.opt, _stream()))


def fm_train_steps(P, Q, bias, ws, bu, bi, bj, batch, first_step, n_steps, hp, adam_step0=0, apply=True, check=True):
    _dev(P, torch.float32, "P"); _dev(Q, torch.float32, "Q"); _dev(bias, torch.float32, "bias")
    for t, nm in ((bu, "bu"), (bi, "bi"), (bj, "bj")):
        _dev(t, torch.int32, nm)
    if bias.numel() != ws.U + ws.I + 1:
        raise ValueError("bias must hold user_num + item_num + 1 floats")
    return _train_steps(L.lib().drb_fm_train_steps, n_steps, P.device, check, _ptr(P), _ptr(Q), _ptr(bias), _ptr(ws.buf), ws.U,
                        ws.I, ws.F, _ptr(bu), _ptr(bi), _ptr(bj), bu.numel(), batch, first_step, n_steps, C.byref(hp), adam_step0,
                        1 if apply else 0)


def fm_rank(P, Q, bias, users, cands, topk):
    _dev(users, torch.int64, "users"); _dev(cands, torch.int64, "cands"); _dev(bias, torch.float32, "bias")
    n, Cn = cands.shape
    out = torch.empty((n, topk), dtype=torch.float32, device=P.device)
    L.check(L.lib().drb_fm_rank(_ptr(P), _ptr(Q), _ptr(bias), P.shape[0], Q.shape[0], P.shape[1], _ptr(users), n, _ptr(cands),
                                Cn, topk, _ptr(out), _stream()))
    return out


def fm_full_rank(P, Q, bias, users, topk):
    _dev(users, torch.int64, "users"); _dev(bias, torch.float32, "bias")
    out = torch.empty((users.numel(), topk), dtype=torch.int64, device=P.device)
    L.check(L.lib().drb_fm_full_rank(_ptr(P), _ptr(Q), _ptr(bias), P.shape[0], Q.shape[0], P.shape[1], _ptr(users),
                                     users.numel(), topk, _ptr(out), _stream()))
    return out


def fm_predict(P, Q, bias, u, i):
    _dev(u, torch.int32, "u"); _dev(i, torch.int32, "i"); _dev(bias, torch.float32, "bias")
    out = torch.empty(u.numel(), dtype=torch.float32, device=P.device)
    L.check(L.lib().drb_fm_predict(_ptr(P), _ptr(Q), _ptr(bias), P.shape[0], Q.shape[0], P.shape[1], _ptr(u), _ptr(i),
                                   u.numel(), _ptr(out), _stream()))
    return out


# ------------------------------------------------------------------ inference
def mf_rank(P, Q, users, cands, topk):
    _dev(users, torch.int64, "users"); _dev(cands, torch.int64, "cands")
    n, Cn = cands.shape
    out = torch.empty((n, topk), dtype=torch.float32, device=P.device)
    L.check(L.lib().drb_mf_rank(_ptr(P), _ptr(Q), P.shape[1], _ptr(users), n, _ptr(cands), Cn, topk, _ptr(out),
                                _stream()))
    return out


def mf_full_rank(P, Q, users, topk):
    _dev(users, torch.int64, "users")
    out = torch.empty((users.numel(), topk), dtype=torch.int64, device=P.device)
    L.check(L.lib().drb_mf_full_rank(_ptr(P), _ptr(Q), P.shape[1], Q.shape[0], _ptr(users), users.numel(), topk,
                                     _ptr(out), _stream()))
    return out


def mf_predict(P, Q, u, i):
    _dev(u, torch.int32, "u"); _dev(i, torch.int32, "i")
    out = torch.empty(u.numel(), dtype=torch.float32, device=P.device)
    L.check(L.lib().drb_mf_predict(_ptr(P), _ptr(Q), P.shape[1], _ptr(u), _ptr(i), u.numel(), _ptr(out), _stream()))
    return out


def mf_rank_host(P, Q, users, cands, topk):
    users = np.ascontiguousarray(users, np.int64)
    cands = np.ascontiguousarray(cands, np.int64)
    out = np.empty((len(users), topk), np.float32)
    L.check(L.lib().drb_mf_rank_host(_ptr(P), _ptr(Q), P.shape[1], users.ctypes.data, len(users), cands.ctypes.data,
                                     cands.shape[1], topk, out.ctypes.data))
    return out


# ------------------------------------------------------------------ LightGCN
def lgcn_norm_adj(coo_u, coo_i, user_num, item_num):
    """get_norm_adj_mat (LightGCNRecommender.py:73-107) as CSR over the U+I nodes, values bit-identical to the
    reference: float64 (deg + 1e-7) ** -0.5, (D*A)*D in float64, cast to fp32.  One-off host build (numpy)."""
    n = user_num + item_num
    u = np.asarray(coo_u, np.int64)
    i = np.asarray(coo_i, np.int64) + user_num
    key = np.unique(np.concatenate([u * n + i, i * n + u]))
    row, col = key // n, key % n
    cnt = np.bincount(row, minlength=n)
    dinv = np.power(cnt.astype(np.float64) + 1e-7, -0.5)
    val = ((dinv[row] * 1.0) * dinv[col]).astype(np.float32)
    row_ptr = np.zeros(n + 1, np.int64)
    np.cumsum(cnt, out=row_ptr[1:])
    return row_ptr, col.astype(np.int32), val


class LgcnGraph:
    """Device copy of the normalised adjacency + its segment list."""

    def __init__(self, row_ptr, col, val, device):
        d_row_ptr = d_col = d_val = None
        if isinstance(row_ptr, torch.Tensor):                    # lgcn_build_adj's device arrays: only the segment
            d_row_ptr, d_col, d_val = row_ptr, col, val          # list is derived on the host (from row_ptr)
            row_ptr = row_ptr.cpu().numpy()
        n = len(row_ptr) - 1
        row_ptr = np.ascontiguousarray(row_ptr, np.int64)
        nseg = int(L.lib().drb_lgcn_segment_count(row_ptr.ctypes.data, n))
        seg_row = np.empty(max(1, nseg), np.int32)
        seg_ptr = np.empty(nseg + 1, np.int64)
        L.check(L.lib().drb_lgcn_segments(row_ptr.ctypes.data, n, seg_row.ctypes.data, seg_ptr.ctypes.data))
        self.n, self.nseg = n, nseg
        if d_row_ptr is not None:
            self.row_ptr, self.col, self.val = d_row_ptr.to(device), d_col.to(device), d_val.to(device)
        else:
            self.row_ptr = torch.from_numpy(row_ptr).to(device)
            self.col = torch.from_numpy(np.ascontiguousarray(col, np.int32)).to(device)
            self.val = torch.from_numpy(np.ascontiguousarray(val, np.float32)).to(device)
        self.seg_row = torch.from_numpy(seg_row).to(device)
        self.seg_ptr = torch.from_numpy(seg_ptr).to(device)
        self.mirror = None

    def args(self):
        return (_ptr(self.row_ptr), _ptr(self.col), _ptr(self.val), _ptr(self.seg_row), _ptr(self.seg_ptr), self.nseg)

    def edge_mirror(self):
        """int32 [nnz]: the CSR slot of (c, r) for every slot (r, c), built once on the device (NGCF's node-dropout backward
        multiplies by the transpose of the dropped adjacency through it).  ValueError when A is not structurally symmetric."""
        if self.mirror is None:
            nnz = int(self.row_ptr[-1].item())
            m = torch.empty(max(nnz, 1), dtype=torch.int32, device=self.row_ptr.device)
            L.check(L.lib().drb_ngcf_edge_mirror(_ptr(self.row_ptr), _ptr(self.col), self.n, nnz, _ptr(m), _stream()))
            if nnz and bool((m[:nnz] < 0).any()):
                raise ValueError("node dropout needs a structurally symmetric adjacency")
            self.mirror = m
        return self.mirror


class LgcnWorkspace:
    def __init__(self, user_num, item_num, factors, opt, device):
        self.U, self.I, self.F = user_num, item_num, factors
        self.opt = L.OPT_SGD if opt == "sgd" else L.OPT_ADAM
        self.buf = torch.empty(L.lib().drb_lgcn_workspace_bytes(user_num, item_num, factors, self.opt), dtype=torch.uint8,
                               device=device)
        L.check(L.lib().drb_lgcn_workspace_init(_ptr(self.buf), user_num, item_num, factors, self.opt, _stream()))


def lgcn_propagate(E0, ws, graph, num_layers, out=None):
    _dev(E0, torch.float32, "E0")
    Em = out if out is not None else torch.empty_like(E0)
    L.check(L.lib().drb_lgcn_propagate(_ptr(E0), _ptr(ws.buf), ws.U, ws.I, ws.F, num_layers, *graph.args(), _ptr(Em),
                                       _stream()))
    return Em


def lgcn_bpr_train_steps(E0, ws, graph, num_layers, bu, bi, bj, batch, first_step, n_steps, hp, adam_step0=0, apply=True,
                         check=True):
    _dev(E0, torch.float32, "E0")
    for t, nm in ((bu, "bu"), (bi, "bi"), (bj, "bj")):
        _dev(t, torch.int32, nm)
    return _train_steps(L.lib().drb_lgcn_bpr_train_steps, n_steps, E0.device, check, _ptr(E0), _ptr(ws.buf), ws.U, ws.I, ws.F,
                        num_layers, *graph.args(), _ptr(bu), _ptr(bi), _ptr(bj), bu.numel(), batch, first_step, n_steps,
                        C.byref(hp), adam_step0, 1 if apply else 0)


# ------------------------------------------------------------------ NGCF
def _dims_arr(dims):
    return (C.c_int32 * len(dims))(*[int(d) for d in dims])


def ngcf_param_count(dims):
    return int(L.lib().drb_ngcf_param_count(_dims_arr(dims), len(dims) - 1))


class NgcfWorkspace:
    def __init__(self, user_num, item_num, dims, opt, device):
        self.U, self.I, self.dims = user_num, item_num, [int(d) for d in dims]
        self.opt = L.OPT_SGD if opt == "sgd" else L.OPT_ADAM
        nbytes = L.lib().drb_ngcf_workspace_bytes(user_num, item_num, _dims_arr(self.dims), len(self.dims) - 1, self.opt)
        if nbytes == 0:
            raise ValueError("NGCF: layer widths must be in 1..256 and 1 <= layers <= 8")
        self.buf = torch.empty(nbytes, dtype=torch.uint8, device=device)
        L.check(L.lib().drb_ngcf_workspace_init(_ptr(self.buf), user_num, item_num, _dims_arr(self.dims), len(self.dims) - 1,
                                                self.opt, _stream()))


def ngcf_keep_bytes(ws):
    """bytes of dropout masks one forward() consumes: one per element of every layer output."""
    return (ws.U + ws.I) * sum(ws.dims[1:])


def ngcf_forward(E0, W, ws, graph, tower_dtype=0, dropout=0.0, keep=None):
    """keep (with mess_dropout > 0): uint8 CUDA tensor, the masks torch's nn.Dropout draws per layer, layers concatenated."""
    _dev(E0, torch.float32, "E0"); _dev(W, torch.float32, "W")
    if keep is not None:
        _dev(keep, torch.uint8, "keep")
        if keep.numel() != ngcf_keep_bytes(ws):
            raise ValueError("keep must hold (user_num + item_num) x sum(hidden widths) bytes")
    out = torch.empty((ws.U + ws.I, sum(ws.dims)), dtype=torch.float32, device=E0.device)
    L.check(L.lib().drb_ngcf_forward(_ptr(E0), _ptr(W), _ptr(ws.buf), ws.U, ws.I, _dims_arr(ws.dims), len(ws.dims) - 1,
                                     *graph.args(), tower_dtype, None if keep is None else _ptr(keep),
                                     C.c_float(dropout if keep is not None else 0.0), _ptr(out), _stream()))
    return out


def ngcf_bpr_train_steps(E0, W, ws, graph, bu, bi, bj, batch, first_step, n_steps, hp, adam_step0=0, apply=True, check=True,
                         tower_dtype=0, dropout=0.0, keep=None):
    _dev(E0, torch.float32, "E0"); _dev(W, torch.float32, "W")
    for t, nm in ((bu, "bu"), (bi, "bi"), (bj, "bj")):
        _dev(t, torch.int32, nm)
    if keep is not None:
        _dev(keep, torch.uint8, "keep")
        if keep.numel() != max(1, n_steps) * ngcf_keep_bytes(ws):
            raise ValueError("keep must hold n_steps x (user_num + item_num) x sum(hidden widths) bytes")
    return _train_steps(L.lib().drb_ngcf_bpr_train_steps, n_steps, E0.device, check, _ptr(E0), _ptr(W), _ptr(ws.buf), ws.U, ws.I,
                        _dims_arr(ws.dims), len(ws.dims) - 1, *graph.args(), _ptr(bu), _ptr(bi), _ptr(bj), bu.numel(), batch,
                        first_step, n_steps, C.byref(hp), adam_step0, 1 if apply else 0, tower_dtype,
                        None if keep is None else _ptr(keep), C.c_float(dropout if keep is not None else 0.0))


def ngcf_forward_philox(E0, W, ws, graph, tower_dtype=0, seed=0, forward=0, mess_dropout=0.0, node_dropout=0.0):
    """forward number ``forward`` with the Philox masks of ``seed``: message dropout, and node dropout when node_dropout > 0."""
    _dev(E0, torch.float32, "E0"); _dev(W, torch.float32, "W")
    out = torch.empty((ws.U + ws.I, sum(ws.dims)), dtype=torch.float32, device=E0.device)
    L.check(L.lib().drb_ngcf_forward_philox(_ptr(E0), _ptr(W), _ptr(ws.buf), ws.U, ws.I, _dims_arr(ws.dims), len(ws.dims) - 1,
                                            *graph.args(), tower_dtype, C.c_uint64(seed), int(forward), C.c_float(mess_dropout),
                                            C.c_double(node_dropout), _ptr(out), _stream()))
    return out


def ngcf_bpr_train_steps_philox(E0, W, ws, graph, bu, bi, bj, batch, first_step, n_steps, hp, adam_step0=0, apply=True,
                                check=True, tower_dtype=0, seed=0, forward0=0, mess_dropout=0.0, node_dropout=0.0):
    """NGCF steps with the Philox masks of ``seed``; step s runs forward number forward0 + s."""
    _dev(E0, torch.float32, "E0"); _dev(W, torch.float32, "W")
    for t, nm in ((bu, "bu"), (bi, "bi"), (bj, "bj")):
        _dev(t, torch.int32, nm)
    mirror = graph.edge_mirror() if node_dropout > 0.0 and apply else None
    return _train_steps(L.lib().drb_ngcf_bpr_train_steps_philox, n_steps, E0.device, check, _ptr(E0), _ptr(W), _ptr(ws.buf), ws.U,
                        ws.I, _dims_arr(ws.dims), len(ws.dims) - 1, *graph.args(), _ptr(bu), _ptr(bi), _ptr(bj), bu.numel(), batch,
                        first_step, n_steps, C.byref(hp), adam_step0, 1 if apply else 0, tower_dtype, C.c_uint64(seed),
                        int(forward0), C.c_float(mess_dropout), C.c_double(node_dropout),
                        None if mirror is None else _ptr(mirror))


def ngcf_philox_masks(seed, forward, user_num, item_num, dims, mess_dropout, node_dropout, nnz, device):
    """test hook: forward number ``forward``'s message masks (uint8, layers concatenated as ``keep``) and edge keep (uint8 [nnz])"""
    dims = [int(d) for d in dims]
    keep = torch.empty((user_num + item_num) * sum(dims[1:]), dtype=torch.uint8, device=device)
    edge = torch.empty(max(int(nnz), 1), dtype=torch.uint8, device=device)
    L.check(L.lib().drb_ngcf_philox_masks(C.c_uint64(seed), int(forward), user_num, item_num, _dims_arr(dims), len(dims) - 1,
                                          C.c_float(mess_dropout), C.c_double(node_dropout), int(nnz), _ptr(keep), _ptr(edge),
                                          _stream()))
    return keep, edge[:int(nnz)]


# ------------------------------------------------------------------ NFM
NFM_ACT = {"relu": 0, "sigmoid": 1, "tanh": 2}


def nfm_param_count(factors, num_layers, batch_norm):
    return int(L.lib().drb_nfm_param_count(factors, num_layers, 1 if batch_norm else 0))


class NfmWorkspace:
    def __init__(self, user_num, item_num, factors, num_layers, batch_norm, opt, max_rows, device):
        self.U, self.I, self.F, self.Ln, self.bn, self.max_rows = user_num, item_num, factors, num_layers, 1 if batch_norm else 0, int(max_rows)
        self.opt = L.OPT_SGD if opt == "sgd" else L.OPT_ADAM
        nbytes = L.lib().drb_nfm_workspace_bytes(user_num, item_num, factors, num_layers, self.bn, self.opt, self.max_rows)
        if nbytes == 0:
            raise ValueError("NFM: factors must be in 1..256, 0 <= num_layers <= 8 and max_rows >= 2")
        self.buf = torch.empty(nbytes, dtype=torch.uint8, device=device)
        L.check(L.lib().drb_nfm_workspace_init(_ptr(self.buf), user_num, item_num, factors, num_layers, self.bn, self.opt,
                                               self.max_rows, _stream()))


def nfm_bpr_train_steps(P, Q, bias, N, Rs, ws, act, bu, bi, bj, batch, first_step, n_steps, hp, adam_step0=0, apply=True,
                        check=True, tower_dtype=0, dropout=0.0, keep=None):
    """keep (with dropout > 0): uint8 CUDA tensor of the masks torch's Dropout modules draw, per step
    [forward call][site][batch][F] (drb_nfm_bpr_train_steps)."""
    for t in (P, Q, bias, N):
        _dev(t, torch.float32, "parameter")
    for t, nm in ((bu, "bu"), (bi, "bi"), (bj, "bj")):
        _dev(t, torch.int32, nm)
    if keep is not None:
        _dev(keep, torch.uint8, "keep")
        rows = batch if n_steps != 1 else min(batch, bu.numel() - first_step * batch)
        if keep.numel() != max(1, n_steps) * 2 * (1 + ws.Ln) * rows * ws.F:
            raise ValueError("keep must hold n_steps x 2 x (1 + num_layers) x batch x factors bytes")
    return _train_steps(
        L.lib().drb_nfm_bpr_train_steps, n_steps, P.device, check, _ptr(P), _ptr(Q), _ptr(bias), _ptr(N),
        None if Rs is None or Rs.numel() == 0 else _ptr(Rs), _ptr(ws.buf), ws.U, ws.I, ws.F, ws.Ln, ws.bn, act, ws.max_rows, _ptr(bu),
        _ptr(bi), _ptr(bj), bu.numel(), batch, first_step, n_steps, C.byref(hp), adam_step0, 1 if apply else 0, tower_dtype,
        None if keep is None else _ptr(keep), C.c_float(dropout if keep is not None else 0.0))


def nfm_bpr_train_steps_philox(P, Q, bias, N, Rs, ws, act, bu, bi, bj, batch, first_step, n_steps, hp, adam_step0=0, apply=True,
                               check=True, tower_dtype=0, dropout=0.0, seed=0):
    """NFM steps with the Dropout masks drawn on the device from Philox: step s keyed by (seed, adam_step0 + s)."""
    for t in (P, Q, bias, N):
        _dev(t, torch.float32, "parameter")
    for t, nm in ((bu, "bu"), (bi, "bi"), (bj, "bj")):
        _dev(t, torch.int32, nm)
    return _train_steps(
        L.lib().drb_nfm_bpr_train_steps_philox, n_steps, P.device, check, _ptr(P), _ptr(Q), _ptr(bias), _ptr(N),
        None if Rs is None or Rs.numel() == 0 else _ptr(Rs), _ptr(ws.buf), ws.U, ws.I, ws.F, ws.Ln, ws.bn, act, ws.max_rows, _ptr(bu),
        _ptr(bi), _ptr(bj), bu.numel(), batch, first_step, n_steps, C.byref(hp), adam_step0, 1 if apply else 0, tower_dtype,
        C.c_float(dropout), C.c_uint64(seed))


def nfm_philox_masks(seed, step, rows, factors, num_layers, dropout, device):
    """test hook: step ``step``'s Philox masks for a batch of ``rows`` triples, uint8 [2 * (1 + num_layers) * rows * factors] in
    the layout of ``keep``"""
    out = torch.empty(2 * (1 + num_layers) * rows * factors, dtype=torch.uint8, device=device)
    L.check(L.lib().drb_nfm_philox_masks(C.c_uint64(seed), int(step), int(rows), factors, num_layers, C.c_float(dropout), _ptr(out),
                                         _stream()))
    return out


def nfm_scores(P, Q, bias, N, Rs, ws, act, u, i, tower_dtype=0):
    """eval-mode scores of the (u[k], i[k]) pairs (int32 CUDA tensors)."""
    _dev(u, torch.int32, "u"); _dev(i, torch.int32, "i")
    out = torch.empty(u.numel(), dtype=torch.float32, device=P.device)
    L.check(L.lib().drb_nfm_scores(_ptr(P), _ptr(Q), _ptr(bias), _ptr(N), None if Rs is None or Rs.numel() == 0 else _ptr(Rs),
                                   _ptr(ws.buf), ws.U, ws.I, ws.F, ws.Ln, ws.bn, act, ws.opt, ws.max_rows, _ptr(u), _ptr(i),
                                   u.numel(), tower_dtype, _ptr(out), _stream()))
    return out


# ------------------------------------------------------------------ NeuMF
NEUMF_MODE = {"NeuMF": 0, "NeuMF-pre": 0, "GMF": 1, "MLP": 2}       # config['model_name'] (NeuMFRecommender.py:48-50)


def neumf_param_count(factors, num_layers, mode=0):
    return int(L.lib().drb_neumf_param_count(factors, num_layers, mode))


def neumf_mask_words(factors, num_layers, batch):
    return int(L.lib().drb_neumf_mask_words(factors, num_layers, batch))


class NeumfWorkspace:
    def __init__(self, user_num, item_num, factors, num_layers, opt, max_rows, device):
        self.U, self.I, self.F, self.Ln, self.max_rows = user_num, item_num, factors, num_layers, int(max_rows)
        self.opt = L.OPT_SGD if opt == "sgd" else L.OPT_ADAM
        nbytes = L.lib().drb_neumf_workspace_bytes(user_num, item_num, factors, num_layers, self.opt, self.max_rows)
        if nbytes == 0:
            raise ValueError("NeuMF: factors must be a positive multiple of 4 and 1 <= num_layers <= 8")
        self.buf = torch.empty(nbytes, dtype=torch.uint8, device=device)
        L.check(L.lib().drb_neumf_workspace_init(_ptr(self.buf), user_num, item_num, factors, num_layers, self.opt,
                                                 self.max_rows, _stream()))


def neumf_bpr_train_steps(tabs, W, ws, bu, bi, bj, batch, first_step, n_steps, hp, adam_step0=0, apply=True, check=True,
                          tower_dtype=0, dropout=0.0, dropout_seed=0, drop_masks=None, mode=0):
    """drop_masks: int32 CUDA tensor [n_steps * neumf_mask_words(F, L, batch)] of host-generated keep-masks (parity mode)."""
    if drop_masks is not None:
        _dev(drop_masks, torch.int32, "drop_masks")
        if drop_masks.numel() < n_steps * neumf_mask_words(ws.F, ws.Ln, batch):
            raise ValueError("drop_masks too short for n_steps batches")
    for t in list(tabs) + [W]:
        _dev(t, torch.float32, "table")
    for t, nm in ((bu, "bu"), (bi, "bi"), (bj, "bj")):
        _dev(t, torch.int32, nm)
    return _train_steps(L.lib().drb_neumf_bpr_train_steps, n_steps, W.device, check, _ptr(tabs[0]), _ptr(tabs[1]), _ptr(tabs[2]),
                        _ptr(tabs[3]), _ptr(W), _ptr(ws.buf), ws.U, ws.I, ws.F, ws.Ln, ws.max_rows, _ptr(bu), _ptr(bi), _ptr(bj),
                        bu.numel(), batch, first_step, n_steps, C.byref(hp), adam_step0, 1 if apply else 0, tower_dtype,
                        C.c_float(dropout), C.c_uint64(dropout_seed), None if drop_masks is None else _ptr(drop_masks), mode)


def neumf_scores(tabs, W, ws, users, items, per_user, tower_dtype=0, mode=0):
    """scores [n_users, per_user]: items = int64 [n_users, per_user] candidate ids, or None for all item ids."""
    _dev(users, torch.int64, "users")
    if items is not None:
        _dev(items, torch.int64, "items")
    out = torch.empty((users.numel(), per_user), dtype=torch.float32, device=W.device)
    L.check(L.lib().drb_neumf_scores(_ptr(tabs[0]), _ptr(tabs[1]), _ptr(tabs[2]), _ptr(tabs[3]), _ptr(W), _ptr(ws.buf), ws.U,
                                     ws.I, ws.F, ws.Ln, ws.opt, ws.max_rows, _ptr(users), users.numel(),
                                     None if items is None else _ptr(items), per_user, tower_dtype, mode, _ptr(out),
                                     _stream()))
    return out


def topk_from_scores(scores, cands, topk):
    _dev(scores, torch.float32, "scores")
    n, cnt = scores.shape
    if cands is not None:
        _dev(cands, torch.int64, "cands")
        out = torch.empty((n, topk), dtype=torch.float32, device=scores.device)
        L.check(L.lib().drb_topk_from_scores(_ptr(scores), _ptr(cands), n, cnt, topk, _ptr(out), None, _stream()))
    else:
        out = torch.empty((n, topk), dtype=torch.int64, device=scores.device)
        L.check(L.lib().drb_topk_from_scores(_ptr(scores), None, n, cnt, topk, None, _ptr(out), _stream()))
    return out


def gemm_test(variant, dtype, A, B, C_out, M, N, K, bias=None, ref=None):
    """Tower GEMM dispatcher (tests): variant 0 NT+bias+ReLU, 1 NN+mask, 2 NN, 3 TN split-K accumulate."""
    L.check(L.lib().drb_gemm_test(variant, dtype, M, N, K, _ptr(A), A.stride(0), _ptr(B), B.stride(0), _ptr(C_out),
                                  C_out.stride(0), None if bias is None else _ptr(bias), None if ref is None else _ptr(ref),
                                  0 if ref is None else ref.stride(0), _stream()))
    return C_out


# ------------------------------------------------------------------ EASE
class EaseX:
    """X of EASERecommender.fit on the device: CSR (row_ptr int64 [U+1], col int32 [nnz], val float32 [nnz]) and the exact-Gram
    scale s (x 2^s are s8 integers), or -1 for the fp64 Gram."""

    def __init__(self, row_ptr, col, val, scale, user_num, item_num):
        self.row_ptr, self.col, self.val, self.scale = row_ptr, col, val, scale
        self.user_num, self.item_num = user_num, item_num


def ease_csr(d_u, d_i, d_v, user_num, item_num):
    """COO (int32 users, int32 items, float64 values) on the device -> EaseX: duplicates summed in fp64 in row order, then
    rounded once to fp32, as csr_matrix((values, (u, i))).astype(float32)."""
    _dev(d_v, torch.float64, "values")
    row_ptr, col = csr_build(d_u, d_i, user_num, item_num)
    seq_ptr, _, order = skipgram_group(d_u, user_num, 0)
    nnz = col.numel()
    val = torch.empty(max(nnz, 1), dtype=torch.float32, device=d_u.device)
    ws = torch.empty(L.lib().drb_ease_csr_workspace_bytes(item_num, nnz), dtype=torch.uint8, device=d_u.device)
    scale = C.c_int32(0)
    L.check(L.lib().drb_ease_csr(_ptr(seq_ptr), _ptr(order), _ptr(d_i), _ptr(d_v), user_num, item_num, _ptr(row_ptr), _ptr(col),
                                 nnz, _ptr(ws), _ptr(val), C.byref(scale), _stream()))
    return EaseX(row_ptr, col.contiguous(), val[:nnz], int(scale.value), user_num, item_num)


def ease_workspace(X, scale=None):
    """Scratch of ease_gram / ease_inverse / ease_weights (the Gram's user-chunk image is sized by the path: X.scale or ``scale``)."""
    s = X.scale if scale is None else scale
    return torch.empty(L.lib().drb_ease_workspace_bytes(X.user_num, X.item_num, s), dtype=torch.uint8, device=X.val.device)


def ease_gram(X, reg, ws, out=None, scale=None):
    """G = X^T X + reg I, fp64 [I, I]: s8 tensor cores when X.scale >= 0 (exact), else fp64 DMMA.  ``scale`` = -1 forces the
    fp64 path (ws must have been sized for it)."""
    s = X.scale if scale is None else scale
    n = X.item_num
    G = torch.empty((n, n), dtype=torch.float64, device=X.val.device) if out is None else _dev(out, torch.float64, "G")
    L.check(L.lib().drb_ease_gram(_ptr(X.row_ptr), _ptr(X.col), _ptr(X.val), X.user_num, n, s, float(reg), _ptr(ws), _ptr(G),
                                  _stream()))
    return G


def ease_inverse(G, ws):
    """In place: G -> G^-1 (blocked sweep on DMMA).  numpy.linalg.LinAlgError when G is not positive definite."""
    _dev(G, torch.float64, "G")
    L.check(L.lib().drb_ease_inverse(_ptr(G), G.shape[0], _ptr(ws), _stream()))
    return G


def ease_weights(P, ws):
    """In place: P -> B = -P / diag(P) (column j divided by P_jj), zero diagonal."""
    _dev(P, torch.float64, "P")
    L.check(L.lib().drb_ease_weights(_ptr(P), P.shape[0], _ptr(ws), _stream()))
    return P


def ease_rank(B, X, users, cands, topk, scores=False):
    """-> int64 [n, topk] candidate item ids by s_c = sum_i x_ui B[c, i] (and the fp64 [n, C] scores when ``scores``)."""
    _dev(B, torch.float64, "B"); _dev(users, torch.int64, "users"); _dev(cands, torch.int64, "cands")
    n, cnum = cands.shape
    out = torch.empty((n, topk), dtype=torch.int64, device=B.device)
    sc = torch.empty((n, cnum), dtype=torch.float64, device=B.device) if scores else None
    L.check(L.lib().drb_ease_rank(_ptr(B), B.shape[0], _ptr(X.row_ptr), _ptr(X.col), _ptr(X.val), _ptr(users), n, _ptr(cands),
                                  cnum, topk, _ptr(out), None if sc is None else _ptr(sc), _stream()))
    return (out, sc) if scores else out


def ease_full_rank(B, X, users, topk, scores=False):
    """-> int64 [n, topk] item ids by s = x_u B (and the fp64 [n, I] scores when ``scores``)."""
    _dev(B, torch.float64, "B"); _dev(users, torch.int64, "users")
    n = users.numel()
    out = torch.empty((n, topk), dtype=torch.int64, device=B.device)
    sc = torch.empty((n, B.shape[0]), dtype=torch.float64, device=B.device)
    L.check(L.lib().drb_ease_full_rank(_ptr(B), B.shape[0], _ptr(X.row_ptr), _ptr(X.col), _ptr(X.val), _ptr(users), n, topk,
                                       _ptr(sc), _ptr(out), _stream()))
    return (out, sc) if scores else out


def ease_predict(B, X, users, items):
    """-> fp64 [n]: x_u . B[:, i] per (u, i) pair."""
    _dev(B, torch.float64, "B"); _dev(users, torch.int64, "users"); _dev(items, torch.int64, "items")
    out = torch.empty(users.numel(), dtype=torch.float64, device=B.device)
    L.check(L.lib().drb_ease_predict(_ptr(B), B.shape[0], _ptr(X.row_ptr), _ptr(X.col), _ptr(X.val), _ptr(users), _ptr(items),
                                     users.numel(), _ptr(out), _stream()))
    return out


# ------------------------------------------------------------------ ItemKNN
# similarity -> (value transform, formula family, ss is the root of the sum of squares): csrc/itemknn.cu.  asymmetric with the
# class's fixed alpha = 0.5 raises ss to the power 1.0 on both sides, which is cosine.
KNN_SIMILARITY = {'cosine': (0, 0, 1), 'asymmetric': (0, 0, 1), 'adjusted': (1, 0, 1), 'pearson': (2, 0, 1),
                  'jaccard': (3, 1, 0), 'tanimoto': (3, 1, 0), 'dice': (3, 2, 0), 'tversky': (3, 3, 0)}


class KnnNeighbours:
    """W of ItemKNNCF by column: idx int32 [I, maxk] (ascending ids, -1 past the count), val float32 [I, maxk], cnt int32 [I]."""

    def __init__(self, idx, val, cnt):
        self.idx, self.val, self.cnt = idx, val, cnt
        self.maxk = idx.shape[1]


def itemknn_transform(X, similarity):
    """The similarity's view of X (KNNCFRecommender.py:165-233, 257-261) -> (EaseX of the transformed values with its own
    exact-Gram scale, ss float32 [I], item_ptr int64 [I+1] of the stored entries per item).  X itself is left as it is."""
    transform, _, root = KNN_SIMILARITY[similarity]
    dev, nnz = X.val.device, X.col.numel()
    item_ptr, _, order = skipgram_group(X.col, X.item_num, 0)
    val = torch.empty(max(nnz, 1), dtype=torch.float32, device=dev)
    ss = torch.empty(X.item_num, dtype=torch.float32, device=dev)
    L.check(L.lib().drb_itemknn_transform(_ptr(X.row_ptr), _ptr(X.val), X.user_num, X.item_num, _ptr(item_ptr), _ptr(order),
                                          transform, root, _ptr(val), _ptr(ss), _stream()))
    ws = torch.empty(L.lib().drb_ease_csr_workspace_bytes(X.item_num, 0), dtype=torch.uint8, device=dev)
    scale = C.c_int32(0)
    L.check(L.lib().drb_ease_scale(_ptr(X.row_ptr), _ptr(X.col), _ptr(val), X.user_num, X.item_num, _ptr(ws), C.byref(scale),
                                   _stream()))
    return EaseX(X.row_ptr, X.col, val[:nnz], int(scale.value), X.user_num, X.item_num), ss, item_ptr


def itemknn_neighbours(G, ss, similarity, normalize, shrink, maxk):
    """compute_similarity's column loop (:302-356) on the Gram matrix G fp64 [n, n] of the transformed values ->
    KnnNeighbours.  Per column the min(maxk, n) largest weights by (weight descending, id ascending), exact zeros dropped."""
    _dev(G, torch.float64, "G"); _dev(ss, torch.float32, "ss")
    n = G.shape[0]
    idx = torch.empty((n, maxk), dtype=torch.int32, device=G.device)
    val = torch.empty((n, maxk), dtype=torch.float32, device=G.device)
    cnt = torch.empty(n, dtype=torch.int32, device=G.device)
    L.check(L.lib().drb_itemknn_neighbours(_ptr(G), n, _ptr(ss), KNN_SIMILARITY[similarity][1], int(bool(normalize)),
                                           float(np.float32(shrink)), maxk, _ptr(idx), _ptr(val), _ptr(cnt), _stream()))
    return KnnNeighbours(idx, val, cnt)


def itemknn_scores(X, W, users, cands=None):
    """pred_mat[u, c] = sum_{i in N(c)} x_ui W[i, c] in fp64 over ascending i -> [n, C] for ``cands`` int64 [n, C], or
    [n, I] over every item."""
    _dev(users, torch.int64, "users")
    n = users.numel()
    cnum = X.item_num if cands is None else _dev(cands, torch.int64, "cands").shape[1]
    sc = torch.empty((n, cnum), dtype=torch.float64, device=users.device)
    L.check(L.lib().drb_itemknn_scores(_ptr(X.row_ptr), _ptr(X.col), _ptr(X.val), _ptr(W.idx), _ptr(W.val), _ptr(W.cnt), W.maxk,
                                       X.item_num, _ptr(users), n, None if cands is None else _ptr(cands), cnum, _ptr(sc),
                                       _stream()))
    return sc


def _itemknn_topk(sc, cands, topk):
    out = torch.empty((sc.shape[0], topk), dtype=torch.int64, device=sc.device)
    L.check(L.lib().drb_itemknn_topk(_ptr(sc), sc.shape[0], sc.shape[1], None if cands is None else _ptr(cands), topk, _ptr(out),
                                     _stream()))
    return out


def itemknn_rank(X, W, users, cands, topk, scores=False):
    """-> int64 [n, topk] candidate ids by (score descending, candidate position ascending) (and the scores when asked)."""
    sc = itemknn_scores(X, W, users, cands)
    out = _itemknn_topk(sc, cands, topk)
    return (out, sc) if scores else out


def itemknn_full_rank(X, W, users, topk, scores=False):
    """-> int64 [n, topk] item ids by (score descending, id ascending) over every item (and the scores when asked)."""
    sc = itemknn_scores(X, W, users)
    out = _itemknn_topk(sc, None, topk)
    return (out, sc) if scores else out


def itemknn_predict(X, W, users, items):
    """-> fp64 [n]: pred_mat[u, i] per (u, i) pair."""
    _dev(items, torch.int64, "items")
    return itemknn_scores(X, W, users, items.reshape(-1, 1)).reshape(-1)


# ------------------------------------------------------------------ UserKNN
USERKNN_PANEL_BYTES = 1 << 32          # the largest Gram panel userknn_neighbours allocates (fp64 [rows, U])


def userknn_transform(X, d_u, d_i, similarity):
    """The similarity's view of X^T [I, U], whose columns are users (KNNCFRecommender.py:491-497) -> (EaseX of X^T with the
    transformed values (rows = items, user_num = I, item_num = U) and its own exact-Gram scale, ss float32 [U]).  adjusted
    removes each item's mean, pearson each user's.  X^T is drb_csr_build of the train COO (d_u, d_i int32) with X's values."""
    transform, _, root = KNN_SIMILARITY[similarity]
    U, I, dev, nnz = X.user_num, X.item_num, X.val.device, X.col.numel()
    t_ptr, t_col = csr_build(d_i, d_u, I, U)
    assert t_col.numel() == nnz
    t_val = torch.empty(max(nnz, 1), dtype=torch.float32, device=dev)
    order = torch.empty(max(nnz, 1), dtype=torch.int32, device=dev)
    L.check(L.lib().drb_userknn_transpose(_ptr(X.row_ptr), _ptr(X.col), _ptr(X.val), U, _ptr(t_ptr), _ptr(t_col), _ptr(t_val),
                                          _ptr(order), _stream()))
    val = torch.empty(max(nnz, 1), dtype=torch.float32, device=dev)
    ss = torch.empty(U, dtype=torch.float32, device=dev)
    L.check(L.lib().drb_itemknn_transform(_ptr(t_ptr), _ptr(t_val), I, U, _ptr(X.row_ptr), _ptr(order), transform, root, _ptr(val),
                                          _ptr(ss), _stream()))
    del t_val, order
    ws = torch.empty(L.lib().drb_ease_csr_workspace_bytes(U, 0), dtype=torch.uint8, device=dev)
    scale = C.c_int32(0)
    L.check(L.lib().drb_ease_scale(_ptr(t_ptr), _ptr(t_col), _ptr(val), I, U, _ptr(ws), C.byref(scale), _stream()))
    return EaseX(t_ptr, t_col.contiguous(), val[:nnz], int(scale.value), I, U), ss


def gram_image(Xt):
    """Dense image of Xt's columns over all of its rows (s8 x 2^scale when Xt.scale >= 0, else fp64) -> uint8 buffer."""
    img = torch.empty(L.lib().drb_gram_image_bytes(Xt.user_num, Xt.item_num, Xt.scale), dtype=torch.uint8, device=Xt.val.device)
    L.check(L.lib().drb_gram_image(_ptr(Xt.row_ptr), _ptr(Xt.col), _ptr(Xt.val), Xt.user_num, Xt.item_num, Xt.scale, _ptr(img),
                                   _stream()))
    return img


def gram_panel(img, Xt, p0, rows, out=None):
    """Rows p0 .. p0 + rows - 1 of Xt^T Xt, fp64 [rows, n] (p0 a multiple of 128), from gram_image(Xt)."""
    n = Xt.item_num
    G = torch.empty((rows, n), dtype=torch.float64, device=img.device) if out is None else out[:rows * n].view(rows, n)
    L.check(L.lib().drb_gram_panel(_ptr(img), Xt.user_num, n, Xt.scale, p0, rows, _ptr(G), _stream()))
    return G


def userknn_panel_rows(user_num, free_bytes):
    """Users per Gram panel: a multiple of 128, at most USERKNN_PANEL_BYTES and ``free_bytes`` of fp64 rows (0: none fits)."""
    cap = min(free_bytes, USERKNN_PANEL_BYTES) // (8 * user_num) // 128 * 128
    return int(min(cap, (user_num + 127) // 128 * 128))


def userknn_neighbours(Xt, ss, similarity, normalize, shrink, maxk, panel):
    """compute_similarity's column loop on X^T: per user column j the min(maxk, U) largest weights by (weight descending, id
    ascending), exact zeros dropped -> KnnNeighbours [U, maxk].  The [U, U] Gram is formed ``panel`` rows at a time (a
    multiple of 128) and each panel's rows are selected before the next is formed."""
    n = Xt.item_num
    if panel <= 0 or panel % 128:
        raise ValueError(f'userknn_neighbours: panel must be a positive multiple of 128, got {panel}')
    dev = Xt.val.device
    idx = torch.empty((n, maxk), dtype=torch.int32, device=dev)
    val = torch.empty((n, maxk), dtype=torch.float32, device=dev)
    cnt = torch.empty(n, dtype=torch.int32, device=dev)
    img = gram_image(Xt)
    rows = min(panel, n)
    buf = torch.empty(rows * n, dtype=torch.float64, device=dev)
    family = KNN_SIMILARITY[similarity][1]
    for p0 in range(0, n, panel):
        r = min(panel, n - p0)
        G = gram_panel(img, Xt, p0, r, buf)
        L.check(L.lib().drb_knn_neighbours_panel(_ptr(G), n, p0, r, _ptr(ss), family, int(bool(normalize)), float(np.float32(shrink)),
                                                 maxk, _ptr(idx), _ptr(val), _ptr(cnt), _stream()))
    return KnnNeighbours(idx, val, cnt)


class KnnReverse:
    """R(u) = {v : u in N(v)} as a CSR over u: r_ptr int64 [U+1], r_col int32 (ascending v), r_val float32 = W[u, v]."""

    def __init__(self, r_ptr, r_col, r_val):
        self.r_ptr, self.r_col, self.r_val = r_ptr, r_col, r_val


def userknn_reverse(W):
    """Forward lists (KnnNeighbours, column v = N(v)) -> KnnReverse."""
    n, maxk = W.idx.shape
    dev = W.idx.device
    pu = torch.empty(n * maxk, dtype=torch.int32, device=dev)
    pv = torch.empty(n * maxk, dtype=torch.int32, device=dev)
    L.check(L.lib().drb_userknn_pairs(_ptr(W.idx), _ptr(W.cnt), n, maxk, _ptr(pu), _ptr(pv), _stream()))
    r_ptr, r_col = csr_build(pu, pv, n + 1, n)
    del pu, pv
    r_ptr = r_ptr[:n + 1].contiguous()
    nnz = int(r_ptr[n].item())
    r_col = r_col[:nnz].contiguous()
    r_val = torch.empty(max(nnz, 1), dtype=torch.float32, device=dev)
    L.check(L.lib().drb_userknn_place(_ptr(W.idx), _ptr(W.val), _ptr(W.cnt), n, maxk, _ptr(r_ptr), _ptr(r_col), _ptr(r_val),
                                      _stream()))
    return KnnReverse(r_ptr, r_col, r_val[:nnz])


def userknn_scores(X, R, users, cands=None):
    """pred_mat[u, c] = sum_{v in R(u)} W[u, v] x_vc in fp64 over ascending v -> [n, C] for ``cands`` int64 [n, C], or [n, I]
    over every item."""
    _dev(users, torch.int64, "users")
    n = users.numel()
    if cands is None:
        sc = torch.empty((n, X.item_num), dtype=torch.float64, device=users.device)
        L.check(L.lib().drb_userknn_full_scores(_ptr(X.row_ptr), _ptr(X.col), _ptr(X.val), _ptr(R.r_ptr), _ptr(R.r_col), _ptr(R.r_val),
                                                X.item_num, _ptr(users), n, _ptr(sc), _stream()))
        return sc
    _dev(cands, torch.int64, "cands")
    sc = torch.empty((n, cands.shape[1]), dtype=torch.float64, device=users.device)
    L.check(L.lib().drb_userknn_scores(_ptr(X.row_ptr), _ptr(X.col), _ptr(X.val), _ptr(R.r_ptr), _ptr(R.r_col), _ptr(R.r_val),
                                       _ptr(users), n, _ptr(cands), cands.shape[1], _ptr(sc), _stream()))
    return sc


def userknn_rank(X, R, users, cands, topk, scores=False):
    """-> int64 [n, topk] candidate ids by (score descending, candidate position ascending) (and the scores when asked)."""
    sc = userknn_scores(X, R, users, cands)
    out = _itemknn_topk(sc, cands, topk)
    return (out, sc) if scores else out


def userknn_full_rank(X, R, users, topk, scores=False):
    """-> int64 [n, topk] item ids by (score descending, id ascending) over every item (and the scores when asked)."""
    sc = userknn_scores(X, R, users)
    out = _itemknn_topk(sc, None, topk)
    return (out, sc) if scores else out


def userknn_predict(X, R, users, items):
    """-> fp64 [n]: pred_mat[u, i] per (u, i) pair."""
    _dev(items, torch.int64, "items")
    return userknn_scores(X, R, users, items.reshape(-1, 1).contiguous()).reshape(-1)


# ------------------------------------------------------------------ MostPop
def mostpop_fit(d_ids, item_num):
    """value_counts of the item ids (int64, every row) -> (cnt fp64 [I], score fp64 [I] = cnt / (1 + cnt)).  IndexError when
    an id is outside [0, item_num)."""
    _dev(d_ids, torch.int64, "ids")
    dev = d_ids.device
    ws = torch.empty(L.lib().drb_mostpop_workspace_bytes(item_num), dtype=torch.uint8, device=dev)
    cnt = torch.empty(item_num, dtype=torch.float64, device=dev)
    score = torch.empty(item_num, dtype=torch.float64, device=dev)
    bad = C.c_int64(0)
    L.check(L.lib().drb_mostpop_fit(_ptr(d_ids), d_ids.numel(), item_num, _ptr(ws), _ptr(cnt), _ptr(score), C.byref(bad), _stream()))
    if bad.value:
        raise IndexError(f'index out of range: {bad.value} item id(s) outside [0, {item_num})')
    return cnt, score


def mostpop_rank(score, cands, topk):
    """-> int64 [n, topk] candidate ids by (score descending, candidate position ascending)."""
    _dev(score, torch.float64, "score"); _dev(cands, torch.int64, "cands")
    sc = torch.empty(cands.shape, dtype=torch.float64, device=cands.device)
    L.check(L.lib().drb_mostpop_gather(_ptr(score), _ptr(cands), cands.numel(), _ptr(sc), _stream()))
    return _itemknn_topk(sc, cands, topk)


def mostpop_order(score, topk):
    """-> int64 [topk] item ids by (score descending, id ascending)."""
    _dev(score, torch.float64, "score")
    return _itemknn_topk(score.view(1, -1), None, topk)[0]


# ------------------------------------------------------------------ SLiM
class SlimPanel:
    """drb_slim_solve's result for targets begin .. begin + count - 1 (row r = item begin + r): the live coordinates lidx int32
    [count, n] (ascending ids, the first nl[r] valid), their coefficients w fp64 and Z = q - G w fp64, and per target the
    sweeps, the unscaled duality gap and whether it converged."""

    def __init__(self, begin, lidx, w, z, nl, sweeps, gap, conv):
        self.begin, self.lidx, self.w, self.z, self.nl = begin, lidx, w, z, nl
        self.sweeps, self.gap, self.conv = sweeps, gap, conv

    def dense(self):
        """-> fp64 [count, n]: each target's full coefficient vector."""
        count, n = self.lidx.shape
        out = torch.zeros((count, n), dtype=torch.float64, device=self.w.device)
        valid = torch.arange(n, device=self.w.device)[None, :] < self.nl[:, None].long()
        rows = torch.arange(count, device=self.w.device)[:, None].expand(count, n)
        out[rows[valid], self.lidx[valid].long()] = self.w[valid]
        return out


def slim_live(G, l1, begin=0, count=None, all_live=False):
    """Items begin .. begin + count - 1 of G fp64 [n, n] = X^T X -> SlimPanel holding each item's live coordinates with w = 0 and
    Z = q (sweeps / gap / conv not yet set).  all_live=False requires every stored value of X to be >= 0 (then coordinates with
    G_kj <= l1, which never leave 0, are skipped exactly)."""
    _dev(G, torch.float64, "G")
    n = G.shape[0]
    count = n - begin if count is None else count
    dev = G.device
    P = max(count, 1)
    diag = torch.empty(n, dtype=torch.float64, device=dev)
    lidx = torch.empty((P, n), dtype=torch.int32, device=dev)
    w = torch.empty((P, n), dtype=torch.float64, device=dev)
    z = torch.empty((P, n), dtype=torch.float64, device=dev)
    nl = torch.empty(P, dtype=torch.int32, device=dev)
    L.check(L.lib().drb_slim_live(_ptr(G), n, begin, count, float(l1), int(bool(all_live)), _ptr(diag), _ptr(lidx), _ptr(w), _ptr(z),
                                  _ptr(nl), _stream()))
    out = SlimPanel(begin, lidx[:count], w[:count], z[:count], nl[:count], None, None, None)
    out.diag = diag
    return out


def slim_solve(G, l1, l2, tol, max_iter, begin=0, count=None, all_live=False, panel=None):
    """SLiMRecommender.py:73-84 for items begin .. begin + count - 1 in Gram form on G fp64 [n, n] = X^T X -> SlimPanel.
    ``panel``: slim_live's result for the same items (built here when None)."""
    P = slim_live(G, l1, begin, count, all_live) if panel is None else panel
    count, n = P.lidx.shape
    dev = G.device
    P.sweeps = torch.empty(max(count, 1), dtype=torch.int32, device=dev)[:count]
    P.gap = torch.empty(max(count, 1), dtype=torch.float64, device=dev)[:count]
    P.conv = torch.empty(max(count, 1), dtype=torch.int32, device=dev)[:count]
    L.check(L.lib().drb_slim_solve(_ptr(G), n, P.begin, count, float(l1), float(l2), float(tol), int(max_iter), _ptr(P.diag),
                                   _ptr(P.lidx), _ptr(P.w), _ptr(P.z), _ptr(P.nl), _ptr(P.sweeps), _ptr(P.gap), _ptr(P.conv),
                                   _stream()))
    return P


def slim_select(panel, topk, out=None):
    """:86-107 for a solved panel -> KnnNeighbours [n, topk] (rows of the panel's items written; pass ``out`` to fill one
    KnnNeighbours panel by panel).  Per item the min(nnz - 1, topk) largest coefficients by (value desc, id asc), fp32."""
    count, n = panel.lidx.shape
    dev = panel.w.device
    if out is None:
        out = KnnNeighbours(torch.full((n, topk), -1, dtype=torch.int32, device=dev), torch.zeros((n, topk), dtype=torch.float32, device=dev),
                            torch.zeros(n, dtype=torch.int32, device=dev))
    L.check(L.lib().drb_slim_select(_ptr(panel.lidx), _ptr(panel.w), _ptr(panel.nl), n, panel.begin, count, topk, _ptr(out.idx),
                                    _ptr(out.val), _ptr(out.cnt), _stream()))
    return out


# ------------------------------------------------------------------ PureSVD
def _round64(x):
    return (x + 63) // 64 * 64


class PureSvdX:
    """X of PureSVD.fit on the device in fp64: the user-major CSR (row_ptr int64 [U+1], col int32 [nnz], val float64 [nnz]) and
    the item-major CSR of X^T (t_ptr int64 [I+1], t_col int32 [nnz] users ascending, t_val float64 [nnz])."""

    def __init__(self, row_ptr, col, val, t_ptr, t_col, t_val, user_num, item_num):
        self.row_ptr, self.col, self.val = row_ptr, col, val
        self.t_ptr, self.t_col, self.t_val = t_ptr, t_col, t_val
        self.user_num, self.item_num = user_num, item_num

    def operand(self, transposed):
        """-> (row_ptr, col, val, n_rows) of X, or of X^T when ``transposed``."""
        if transposed:
            return self.t_ptr, self.t_col, self.t_val, self.item_num
        return self.row_ptr, self.col, self.val, self.user_num


def puresvd_csr(d_u, d_i, d_v, user_num, item_num):
    """COO (int32 users, int32 items, float64 values) on the device -> PureSvdX: duplicates summed in fp64 in row order, as
    csr_matrix((values, (u, i)), (U, I)) up to the order scipy gives three or more duplicates of one pair."""
    _dev(d_v, torch.float64, "values")
    row_ptr, col = csr_build(d_u, d_i, user_num, item_num)
    col = col.contiguous()
    seq_ptr, _, order = skipgram_group(d_u, user_num, 0)
    t_ptr, t_col = csr_build(d_i, d_u, item_num, user_num)
    nnz, dev = col.numel(), d_u.device
    assert t_col.numel() == nnz
    t_col = t_col.contiguous()
    val = torch.empty(max(nnz, 1), dtype=torch.float64, device=dev)
    t_val = torch.empty(max(nnz, 1), dtype=torch.float64, device=dev)
    L.check(L.lib().drb_puresvd_csr(_ptr(seq_ptr), _ptr(order), _ptr(d_i), _ptr(d_v), user_num, item_num, _ptr(row_ptr), _ptr(col),
                                    nnz, _ptr(t_ptr), _ptr(t_col), _ptr(val), _ptr(t_val), _stream()))
    return PureSvdX(row_ptr, col, val[:nnz], t_ptr, t_col, t_val[:nnz], user_num, item_num)


def puresvd_panel(rows, l, device):
    """A zero fp64 panel [rows rounded up to 64, l rounded up to 64] (the layout of every PureSVD panel)."""
    return torch.zeros((_round64(rows), _round64(l)), dtype=torch.float64, device=device)


def puresvd_spmm(A, Z, l, Y):
    """Y[r, :l] = sum_j A[r, j] Z[j, :l] for A = (row_ptr, col, val, n_rows); Y's columns l .. ld are written 0."""
    row_ptr, col, val, n_rows = A
    _dev(Z, torch.float64, "Z"); _dev(Y, torch.float64, "Y")
    L.check(L.lib().drb_puresvd_spmm(_ptr(row_ptr), _ptr(col), _ptr(val), n_rows, _ptr(Z), l, Y.shape[1], _ptr(Y), _stream()))
    return Y


def puresvd_orth_workspace(m, l, device):
    return torch.empty(L.lib().drb_puresvd_orth_workspace_bytes(m, _round64(l)), dtype=torch.uint8, device=device)


def puresvd_orth(Y, m, l, ws=None, want_r=False):
    """In place: the first m rows of the panel Y -> Q of shifted CholeskyQR3 (Y = Q R).  -> R fp64 [ld, ld] (upper, padded block
    identity) when ``want_r``.  numpy.linalg.LinAlgError when the panel is numerically rank deficient."""
    _dev(Y, torch.float64, "Y")
    ld = Y.shape[1]
    ws = puresvd_orth_workspace(m, l, Y.device) if ws is None else ws
    R = torch.empty((ld, ld), dtype=torch.float64, device=Y.device) if want_r else None
    L.check(L.lib().drb_puresvd_orth(_ptr(Y), m, l, ld, _ptr(ws), None if R is None else _ptr(R), _stream()))
    return R


def puresvd_small_svd(R, l):
    """One-sided Jacobi SVD of R[:l, :l]^T -> (s fp64 [l], UT fp64 [ld, ld], VT fp64 [ld, ld]): rows j of UT / VT are the left /
    right singular vectors of R^T for s[j], unsorted."""
    _dev(R, torch.float64, "R")
    ld = R.shape[1]
    s = torch.empty(l, dtype=torch.float64, device=R.device)
    UT = torch.empty((ld, ld), dtype=torch.float64, device=R.device)
    VT = torch.empty((ld, ld), dtype=torch.float64, device=R.device)
    L.check(L.lib().drb_puresvd_small_svd(_ptr(R), l, ld, _ptr(s), _ptr(UT), _ptr(VT), _stream()))
    return s, UT, VT


def puresvd_factors(Q, m, Qb, n, l, s, UT, VT, transposed, k, user_num, item_num):
    """U_A = Q Ur, V_A = Q_b Vr for the k largest sigma -> (user_vec fp64 [U, k], item_vec fp64 [I, k], sigma fp64 [l] sorted)."""
    ld = Q.shape[1]
    dev = Q.device
    ws = torch.empty(L.lib().drb_puresvd_factors_workspace_bytes(m, n, ld, k), dtype=torch.uint8, device=dev)
    P = torch.empty((user_num, k), dtype=torch.float64, device=dev)
    V = torch.empty((item_num, k), dtype=torch.float64, device=dev)
    sigma = torch.empty(l, dtype=torch.float64, device=dev)
    L.check(L.lib().drb_puresvd_factors(_ptr(Q), m, _ptr(Qb), n, l, ld, _ptr(s), _ptr(UT), _ptr(VT), int(bool(transposed)), k,
                                        _ptr(ws), _ptr(P), _ptr(V), _ptr(sigma), _stream()))
    return P, V, sigma


def puresvd_fit(X, omega, factors, n_iter, transposed, mark=None):
    """randomized_svd's sequence on the device: Omega (host fp64 [min(U, I), l]) -> n_iter rounds of Y = orth(A Z),
    Z = orth(A^T Y), then Q = orth(A Z), Q_b R = A^T Q, the SVD of R^T and the factors.  A = X^T when ``transposed``.
    ``mark(phase)`` is called after each phase (for timing).  -> (user_vec, item_vec, sigma)."""
    dev = X.val.device
    mark = mark or (lambda phase: None)
    n, l = omega.shape
    A, At = X.operand(transposed), X.operand(not transposed)
    m = A[3]
    Z = puresvd_panel(n, l, dev)
    Z[:n, :l] = torch.from_numpy(np.ascontiguousarray(omega, np.float64)).to(dev)
    Y = puresvd_panel(m, l, dev)
    ws_m, ws_n = puresvd_orth_workspace(m, l, dev), puresvd_orth_workspace(n, l, dev)
    mark("upload")
    for _ in range(n_iter):
        puresvd_spmm(A, Z, l, Y); mark("spmm")
        puresvd_orth(Y, m, l, ws_m); mark("orth")
        puresvd_spmm(At, Y, l, Z); mark("spmm")
        puresvd_orth(Z, n, l, ws_n); mark("orth")
    puresvd_spmm(A, Z, l, Y); mark("spmm")
    puresvd_orth(Y, m, l, ws_m); mark("orth")
    puresvd_spmm(At, Y, l, Z); mark("spmm")
    R = puresvd_orth(Z, n, l, ws_n, want_r=True); mark("orth")
    del ws_m, ws_n
    s, UT, VT = puresvd_small_svd(R, l); mark("small_svd")
    out = puresvd_factors(Y, m, Z, n, l, s, UT, VT, transposed, factors, X.user_num, X.item_num); mark("factors")
    return out


def puresvd_scores(user_vec, item_vec, users, cands=None):
    """-> fp64 [n, C] user_vec[u] . item_vec[c] for ``cands`` int64 [n, C], or [n, I] over every item."""
    _dev(user_vec, torch.float64, "user_vec"); _dev(item_vec, torch.float64, "item_vec"); _dev(users, torch.int64, "users")
    n, k = users.numel(), user_vec.shape[1]
    cnum = item_vec.shape[0] if cands is None else _dev(cands, torch.int64, "cands").shape[1]
    sc = torch.empty((n, cnum), dtype=torch.float64, device=users.device)
    L.check(L.lib().drb_puresvd_scores(_ptr(user_vec), _ptr(item_vec), k, _ptr(users), n, None if cands is None else _ptr(cands),
                                       cnum, _ptr(sc), _stream()))
    return sc


def puresvd_rank(user_vec, item_vec, users, cands, topk, scores=False):
    """-> int64 [n, topk] candidate ids by (score descending, candidate position ascending) (and the scores when asked)."""
    sc = puresvd_scores(user_vec, item_vec, users, cands)
    out = _itemknn_topk(sc, cands, topk)
    return (out, sc) if scores else out


def puresvd_full_rank(user_vec, item_vec, users, topk, scores=False):
    """-> int64 [n, topk] item ids by (score descending, id ascending) over every item (and the scores when asked)."""
    sc = puresvd_scores(user_vec, item_vec, users)
    out = _itemknn_topk(sc, None, topk)
    return (out, sc) if scores else out


def puresvd_predict(user_vec, item_vec, users, items):
    """-> fp64 [n]: user_vec[u] . item_vec[i] per (u, i) pair."""
    _dev(items, torch.int64, "items")
    return puresvd_scores(user_vec, item_vec, users, items.reshape(-1, 1).contiguous()).reshape(-1)


# ------------------------------------------------------------------ Multi-VAE
def _vae_hidden(hidden):
    return (C.c_int32 * max(1, len(hidden)))(*[int(h) for h in hidden]), len(hidden)


def vae_param_count(item_num, hidden, latent_dim):
    h, nh = _vae_hidden(hidden)
    return int(L.lib().drb_vae_param_count(item_num, h, nh, latent_dim))


class VaeInput:
    """The input rows of every user (drb_vae_input_csr): row_ptr int64 [U + 1], col int32 / val fp32 [nnz] on the device."""

    def __init__(self, hist_id, hist_val, item_num):
        _dev(hist_id, torch.int64, "history_item_id")
        _dev(hist_val, torch.float32, "history_item_value")
        U, Lh = hist_id.shape
        self.user_num, self.item_num = int(U), int(item_num)
        self.row_ptr = torch.empty(U + 1, dtype=torch.int64, device=hist_id.device)
        nnz = C.c_int64()
        L.check(L.lib().drb_vae_input_csr(_ptr(hist_id), _ptr(hist_val), U, Lh, item_num, _ptr(self.row_ptr), None, None,
                                          C.byref(nnz), _stream()))
        self.col = torch.empty(max(1, nnz.value), dtype=torch.int32, device=hist_id.device)
        self.val = torch.empty(max(1, nnz.value), dtype=torch.float32, device=hist_id.device)
        L.check(L.lib().drb_vae_input_csr(_ptr(hist_id), _ptr(hist_val), U, Lh, item_num, _ptr(self.row_ptr), _ptr(self.col),
                                          _ptr(self.val), C.byref(nnz), _stream()))
        self.nnz = nnz.value
        self.max_row_len = int((self.row_ptr[1:] - self.row_ptr[:-1]).max().item())


VAE_MAX_ROWS = 32768       # users per step / scoring pass (drb_vae_train_steps)


class VaeWorkspace:
    """opt: 'sgd' / 'adam', or None for a scoring workspace (no gradient or optimiser state).  The nonzero scratch holds
    max_rows rows of the input's longest row, so no batch of at most max_rows users outgrows it."""

    def __init__(self, item_num, hidden, latent_dim, opt, max_rows, max_row_len, device):
        self.I, self.hidden, self.lat = int(item_num), [int(h) for h in hidden], int(latent_dim)
        self.max_rows, self.max_row_len = int(max_rows), int(max_row_len)
        if not 1 <= self.max_rows <= VAE_MAX_ROWS:
            raise ValueError(f"Multi-VAE: a step takes 1 .. {VAE_MAX_ROWS} users, got {self.max_rows}")
        self.opt = -1 if opt is None else (L.OPT_SGD if opt == "sgd" else L.OPT_ADAM)
        self._h = _vae_hidden(self.hidden)
        nbytes = L.lib().drb_vae_workspace_bytes(self.I, *self._h, self.lat, self.opt, self.max_rows, self.max_row_len)
        if nbytes == 0:
            raise ValueError("Multi-VAE: need 1 <= item_num <= 2^20, at most 8 positive hidden sizes and latent_dim >= 2")
        self.buf = torch.empty(nbytes, dtype=torch.uint8, device=device)
        L.check(L.lib().drb_vae_workspace_init(_ptr(self.buf), self.I, *self._h, self.lat, self.opt, self.max_rows,
                                               self.max_row_len, _stream()))

    def state_bytes(self):
        """bytes of the header, gradient and optimiser state at the start of the workspace (the library's carve)"""
        a = lambda n: (n + 255) // 256 * 256  # noqa: E731
        nW = vae_param_count(self.I, self.hidden, self.lat)
        return 256 + {-1: 0, L.OPT_SGD: 1, L.OPT_ADAM: 3}[self.opt] * a(4 * nW)

    def grown(self, max_rows):
        """a workspace for up to max_rows users carrying this one's gradient and optimiser state"""
        new = VaeWorkspace(self.I, self.hidden, self.lat, {-1: None, L.OPT_SGD: "sgd", L.OPT_ADAM: "adam"}[self.opt],
                           max_rows, self.max_row_len, self.buf.device)
        n = self.state_bytes()
        new.buf[:n].copy_(self.buf[:n])
        return new

    def dims(self):
        return (self.I, *self._h, self.lat, self.opt, self.max_rows, self.max_row_len)


def vae_keep_words(batch, item_num):
    """uint32 words of one step's bit-packed [batch, item_num] keep mask."""
    return (batch * item_num + 31) // 32


def vae_train_steps(W, ws, inp, users, batch, first_step, n_steps, hp, adam_step0=0, apply=True, training=True, update0=0,
                    total_anneal_steps=0, anneal_cap=0.2, dropout=0.0, seed=0, keep_bits=None, eps=None, check=True):
    """users: int64 CUDA tensor of the epoch's batch rows; keep_bits (int32 [n_steps * vae_keep_words]) and eps (fp32
    [n_steps, batch, latent_dim // 2]): host draws, both or neither (drb_vae_train_steps)."""
    _dev(W, torch.float32, "W")
    _dev(users, torch.int64, "users")
    if (keep_bits is None) != (eps is None) and training and dropout > 0.0:
        raise ValueError("keep_bits and eps are drawn together")
    if keep_bits is not None:
        _dev(keep_bits, torch.int32, "keep_bits")
        if keep_bits.numel() < n_steps * vae_keep_words(batch, ws.I):
            raise ValueError("keep_bits too short for n_steps batches")
    if eps is not None:
        _dev(eps, torch.float32, "eps")
        if eps.numel() < n_steps * batch * (ws.lat // 2):
            raise ValueError("eps too short for n_steps batches")
    return _train_steps(
        L.lib().drb_vae_train_steps, n_steps, W.device, check, _ptr(W), _ptr(ws.buf), *ws.dims(), _ptr(inp.row_ptr),
        _ptr(inp.col), _ptr(inp.val), _ptr(users), users.numel(), batch, first_step, n_steps, C.byref(hp), adam_step0,
        1 if apply else 0, 1 if training else 0, int(update0), int(total_anneal_steps), C.c_double(anneal_cap),
        C.c_float(dropout), C.c_uint64(seed), None if keep_bits is None else _ptr(keep_bits), None if eps is None else _ptr(eps))


def vae_scores(W, ws, inp, users, cands=None):
    """eval-mode logits: [n, C] of the candidates (int64 [n, C]) or [n, item_num] of every item."""
    _dev(users, torch.int64, "users")
    if cands is not None:
        _dev(cands, torch.int64, "cands")
    n, cnt = users.numel(), (cands.shape[1] if cands is not None else ws.I)
    out = torch.empty((n, cnt), dtype=torch.float32, device=W.device)
    L.check(L.lib().drb_vae_scores(_ptr(W), _ptr(ws.buf), *ws.dims(), _ptr(inp.row_ptr), _ptr(inp.col), _ptr(inp.val),
                                   _ptr(users), n, None if cands is None else _ptr(cands), cnt, _ptr(out), _stream()))
    return out


def vae_philox_draws(seed, step, dropout, rows, cols, half, device):
    """test hook: the 'philox' engine's keep bits uint8 [rows, cols] and normals fp32 [rows, half] of one step"""
    keep = torch.empty((rows, cols), dtype=torch.uint8, device=device)
    eps = torch.empty((rows, half), dtype=torch.float32, device=device)
    L.check(L.lib().drb_vae_philox_draws(C.c_uint64(seed), step, C.c_float(dropout), rows, cols, half, _ptr(keep), _ptr(eps),
                                         _stream()))
    return keep, eps
