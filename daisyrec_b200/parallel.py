"""User-sharded multi-GPU BPR-MF (one process per GPU, SURVEY.md section 8(e)).

The reference has no multi-device path at all (single process, `AbstractRecommender.py:99-100`), so the
single-GPU run of this framework is the oracle for N > 1:

* the USER table is row-sharded by contiguous user ranges balanced by interaction count; rank r owns the
  rows and every training triple of its users -- user-row reads and updates are always local;
* the ITEM table (<= 9 MB at every BASELINE shape) is replicated;
* every rank walks the same global epoch permutation and keeps the triples of its users
  (`drb_shard_gather_triples`), so the union of the local batches of step s IS the single-GPU batch s;
* per step: phase 1 on the local triples -> NCCL all-reduce (sum) of the item-gradient accumulator, the item
  counters and the 8 loss/norm scalars -> phase 2 (local user rows + the full item table, bit-identically on
  every rank because the reduced inputs are identical);
* at rank time each GPU scores its own users and ONE all-gather assembles the per-user top-K in loader order.

torch.distributed (NCCL on GPUs, gloo in the CPU tests of the host logic) is plumbing; all compute is in
libdaisyrec_b200.so.
"""
import ctypes as C
import os
import numpy as np
import torch
import torch.distributed as dist

from . import _lib as L


# --------------------------------------------------------------------------------------- host logic
def partition_users(weights, world):
    """Contiguous user ranges with ~equal total weight (interaction / triple counts).

    weights: int array [U] (non-negative).  Returns int64 bounds[world+1], bounds[0]=0, bounds[-1]=U;
    rank r owns users [bounds[r], bounds[r+1])."""
    w = np.asarray(weights, dtype=np.int64)
    U = len(w)
    csum = np.concatenate([[0], np.cumsum(w)])
    total = int(csum[-1])
    bounds = np.zeros(world + 1, np.int64)
    for r in range(1, world):
        target = (total * r + world - 1) // world
        bounds[r] = int(np.searchsorted(csum, target, side="left"))
    bounds[world] = U
    return np.maximum.accumulate(np.minimum(bounds, U))


def owner_of(users, bounds):
    """Rank owning each user id."""
    return np.searchsorted(np.asarray(bounds)[1:], np.asarray(users), side="right")


def allreduce_step_buffers(gq, cnt_i, acc, group=None):
    """The per-step exchange: item-gradient accumulator (fp32), item counters (int64 view of the packed
    u64 pos|neg<<32 pairs: the halves never carry into each other below 2^32 occurrences), and the 8 fp64
    loss / norm partial sums."""
    dist.all_reduce(gq, op=dist.ReduceOp.SUM, group=group)
    dist.all_reduce(cnt_i, op=dist.ReduceOp.SUM, group=group)
    dist.all_reduce(acc, op=dist.ReduceOp.SUM, group=group)


def allgather_rows(local_rows, local_pos, total_rows, group=None):
    """Assemble a [total_rows, K] matrix from per-rank row blocks with ONE all-gather.

    local_rows: [n_local, K] tensor; local_pos: int64 [n_local] destination row of each local row.
    Variable counts are padded to the maximum (all_gather needs equal shapes); position -1 marks padding."""
    world = dist.get_world_size(group)
    n_local = torch.tensor([local_rows.shape[0]], dtype=torch.int64, device=local_rows.device)
    counts = [torch.zeros_like(n_local) for _ in range(world)]
    dist.all_gather(counts, n_local, group=group)
    n_max = max(int(c.item()) for c in counts)
    K = local_rows.shape[1]
    # pack positions next to the payload so a single collective moves both
    payload = torch.full((n_max, K + 1), -1, dtype=torch.float64, device=local_rows.device)
    payload[:local_rows.shape[0], :K] = local_rows.to(torch.float64)
    payload[:local_rows.shape[0], K] = local_pos.to(torch.float64)
    gathered = [torch.empty_like(payload) for _ in range(world)]
    dist.all_gather(gathered, payload, group=group)
    out = torch.zeros((total_rows, K), dtype=local_rows.dtype, device=local_rows.device)
    for g in gathered:
        pos = g[:, K].to(torch.int64)
        keep = pos >= 0
        out[pos[keep]] = g[keep, :K].to(local_rows.dtype)
    return out


def broadcast_cpu_(t, device, group=None):
    """In-place broadcast of a CPU tensor from rank 0 (staged through `device` when the backend is NCCL)."""
    if dist.get_backend(group) == "nccl":
        d = t.to(device)
        dist.broadcast(d, 0, group=group)
        t.copy_(d)
    else:
        dist.broadcast(t, 0, group=group)
    return t


def broadcast_int(value, device, group=None):
    """Rank 0's python int on every rank (seeds, sizes)."""
    t = torch.tensor([int(value)], dtype=torch.int64)
    return int(broadcast_cpu_(t, device, group).item())


# --------------------------------------------------------------------------------------- device side
_NATIVE_COMM = {"ready": False}


def init_native_comm(group=None):
    """Create the library's own NCCL communicator (rank 0's ncclUniqueId is broadcast with torch.distributed)."""
    if _NATIVE_COMM["ready"]:
        return
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    ident = torch.zeros(128, dtype=torch.uint8, device="cuda")
    if rank == 0:
        buf = (C.c_uint8 * 128)()
        L.check(L.lib().drb_comm_unique_id(buf))
        ident.copy_(torch.tensor(list(buf), dtype=torch.uint8))
    dist.broadcast(ident, 0, group=group)
    host = ident.cpu().numpy()
    L.check(L.lib().drb_comm_init(host.ctypes.data, rank, world))
    _NATIVE_COMM["ready"] = True


_HOST_GROUP = {}


def _host_group(group=None):
    """A gloo (host-only) group over the same ranks, for barriers that must not occupy the GPUs.  Collective on first use."""
    key = id(group)
    if key not in _HOST_GROUP:
        ranks = None if group is None else dist.get_process_group_ranks(group)
        if os.environ.get("MASTER_ADDR", "127.0.0.1") in ("127.0.0.1", "localhost"):
            os.environ.setdefault("GLOO_SOCKET_IFNAME", "lo")   # one node: no hostname resolution (it may not resolve in a container)
        _HOST_GROUP[key] = dist.new_group(ranks=ranks, backend="gloo")
    return _HOST_GROUP[key]


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return C.c_void_p(t.data_ptr())


class ShardedTrainer:
    """Rank-local state of user-sharded BPR-MF training."""

    def __init__(self, P_local, Q, bounds, rank, world, hp, opt="sgd", group=None, comm="nccl"):
        from . import ops
        if comm == "auto":
            # the peer-exchange kernel is the default where it has been validated on hardware (2 GPUs: parity + 0.91 weak-scaling
            # efficiency); larger worlds take the NCCL step unless 'p2p' is asked for by name (DESIGN.md, multi-GPU section)
            comm = "p2p" if world == 2 else "nccl"
        # comm = "nccl": the library enqueues kernels + one grouped NCCL all-reduce per step itself (no host round trip);
        # comm = "torch": per-step torch.distributed collectives (also what the gloo CPU tests of the host logic exercise)
        # comm = "p2p": ONE persistent launch per epoch segment, the exchange inside the kernel over peer-mapped memory (csrc/p2p.cu)
        self.comm = comm if (comm == "torch" or dist.get_backend(group) == "nccl") else "torch"
        if self.comm == "p2p" and (hp.opt not in (L.OPT_SGD, L.OPT_ADAM) or hp.loss != 0 or Q.shape[1] % 4 or Q.shape[1] > 128
                                   or world > 8):
            self.comm = "nccl"                                    # outside the peer kernel's instantiations
        if self.comm == "nccl":
            init_native_comm(group)
        if self.comm in ("nccl", "p2p"):
            ops.mf_step_variant(Q.shape[1], P_local.shape[0] + Q.shape[0])   # the step kernel's one-off on-device selection, before any peer waits on us
        self.ops = ops
        self.Q = Q
        self._xbuf = None
        if self.comm == "p2p":
            self._open_peer_buffers(Q, rank, world, group)
        # a rank that owns no user still takes part in every collective: give the kernels one dummy row to point at
        self.P = P_local if P_local.shape[0] > 0 else torch.zeros((1, Q.shape[1]), dtype=Q.dtype, device=Q.device)
        self.bounds, self.rank, self.world, self.group = np.asarray(bounds, np.int64), rank, world, group
        self.lo, self.hi = int(self.bounds[rank]), int(self.bounds[rank + 1])
        self.U_local, self.I, self.F = P_local.shape[0], Q.shape[0], Q.shape[1]
        assert self.U_local == self.hi - self.lo
        self.hp = hp
        self.dev = Q.device
        self.ws = ops.MFWorkspace(max(1, self.U_local), self.I, self.F, opt, self.dev)
        lay = (C.c_int64 * 8)()
        L.check(L.lib().drb_mf_workspace_layout(max(1, self.U_local), self.I, self.F, self.ws.opt, lay))
        buf = self.ws.buf
        self.acc = buf[lay[0]:lay[0] + lay[1]].view(torch.float64)
        self.gq = buf[lay[2]:lay[2] + lay[3]].view(torch.float32)
        self.cnt_i = buf[lay[4]:lay[4] + lay[5]].view(torch.int64)
        self.loss = torch.zeros(1, dtype=torch.float64, device=self.dev)
        self.opt_steps = 0
        self.offsets_host = None
        self._stage = None
        self.peer_timeout_s = 20.0

    # ---- peer exchange buffers (comm = "p2p")
    def _open_peer_buffers(self, Q, rank, world, group):
        I, F = Q.shape
        lib = L.lib()
        nbytes = lib.drb_p2p_buffer_bytes(I, F)
        own, handle = C.c_void_p(), (C.c_uint8 * 64)()
        L.check(lib.drb_p2p_alloc(nbytes, C.byref(own), handle))
        self._xbuf, self._xbytes = own.value, nbytes
        mine = torch.tensor(list(handle), dtype=torch.uint8, device=Q.device)
        every = [torch.empty_like(mine) for _ in range(world)]
        dist.all_gather(every, mine, group=group)                  # torch.distributed moves the 64-byte handles, nothing else
        handles = [e.cpu().tolist() for e in every]
        torch.cuda.synchronize()
        self._peer_ptrs = (C.c_void_p * world)()
        self._opened = []
        # Mapping a peer's buffer creates / touches a context on the peer's device.  The ranks take turns, separated by a HOST
        # barrier (gloo), with every GPU idle: no rank sits in a device-side collective while another one maps its memory.
        hg = _host_group(group)
        for turn in range(world):
            if turn == rank:
                for q in range(world):
                    if q == rank:
                        self._peer_ptrs[q] = own.value
                        continue
                    h = (C.c_uint8 * 64)(*handles[q])
                    ptr = C.c_void_p()
                    L.check(lib.drb_p2p_open(h, C.byref(ptr)))
                    self._peer_ptrs[q] = ptr.value
                    self._opened.append(ptr.value)
            dist.barrier(group=hg)
        # the item-table replica lives inside the exchange buffer (peers store their slices straight into it)
        q_off = lib.drb_p2p_q_offset(I, F)

        class _Mem:
            __cuda_array_interface__ = {"shape": (I * F,), "typestr": "<f4", "data": (own.value + q_off, False), "version": 2}
        self._q_owner = _Mem()
        q_view = torch.as_tensor(self._q_owner, device=Q.device).view(I, F)
        q_view.copy_(Q)
        self.Q = q_view
        torch.cuda.synchronize()
        dist.barrier(group=group)                                  # every replica is initialised before anyone's first launch

    def close(self):
        """Unmap the peers' buffers and free the own one (collective: nobody may still be inside a launch)."""
        if self._xbuf is None:
            return
        torch.cuda.synchronize()
        hg = _host_group(self.group)
        dist.barrier(group=hg)                                     # host barriers: the GPUs stay idle while mappings change
        q_copy = self.Q.clone()
        torch.cuda.synchronize()
        for turn in range(self.world):
            if turn == self.rank:
                for ptr in self._opened:
                    L.lib().drb_p2p_close(C.c_void_p(ptr))
            dist.barrier(group=hg)
        L.lib().drb_p2p_free(C.c_void_p(self._xbuf))
        self._xbuf, self._opened, self.Q = None, [], q_copy

    # ---- train feed
    def prepare_epoch(self, d_triples, d_perm, batch_global):
        """Local SoA planes + per-step offsets from the global permutation."""
        n = d_triples.shape[0] if d_perm is None else d_perm.numel()
        m = (n + batch_global - 1) // batch_global
        # upper bound of local triples: count once (cheap) via the counting pass inside the library
        self.scratch = torch.empty(max(1, m), dtype=torch.int64, device=self.dev)
        self.step_offsets = torch.empty(m + 1, dtype=torch.int64, device=self.dev)
        cap = n                                                   # worst case; planes are views of one buffer
        if getattr(self, "_planes", None) is None or self._planes.shape[1] < cap:
            self._planes = torch.empty((3, (cap + 3) // 4 * 4), dtype=torch.int32, device=self.dev)
        L.check(L.lib().drb_shard_gather_triples(_ptr(d_triples), None if d_perm is None else _ptr(d_perm), n, self.lo,
                                                 self.hi, batch_global, _ptr(self.scratch), _ptr(self.step_offsets),
                                                 _ptr(self._planes[0]), _ptr(self._planes[1]), _ptr(self._planes[2]),
                                                 _stream()))
        self.offsets_host = self.step_offsets.cpu().numpy()
        self.batch_global = int(batch_global)
        self.bu, self.bi, self.bj = self._planes[0], self._planes[1], self._planes[2]
        if self.comm == "p2p":
            # everything a launch needs is allocated here, and every rank has finished allocating before anyone can sit in a
            # launch waiting for its peers (a device allocation in one process may have to touch its peers' mappings)
            if getattr(self, "_losses", None) is None or self._losses.numel() < m + 1:
                self._losses = torch.empty(m + 1, dtype=torch.float64, device=self.dev)
            torch.cuda.synchronize()
            dist.barrier(group=_host_group(self.group))
        return m

    # ---- one synchronous global step
    def _phase(self, phase, bu, bi, bj, begin, count):
        L.check(L.lib().drb_mf_bpr_phase(_ptr(self.P), _ptr(self.Q), _ptr(self.ws.buf), max(1, self.U_local), self.I, self.F,
                                         _ptr(bu), _ptr(bi), _ptr(bj), begin, count, phase, C.byref(self.hp),
                                         self.opt_steps, _ptr(self.loss), _stream()))

    def step_device(self, bu, bi, bj, begin, count):
        self._phase(1, bu, bi, bj, begin, count)
        allreduce_step_buffers(self.gq, self.cnt_i, self.acc, self.group)
        self._phase(2, bu, bi, bj, begin, count)
        self.opt_steps += 1

    def step(self, s):
        b, e = int(self.offsets_host[s]), int(self.offsets_host[s + 1])
        self.step_device(self.bu, self.bi, self.bj, b, e - b)

    def train_steps(self, first, n_steps, losses=None):
        """Global steps first .. first+n_steps-1 of the prepared epoch; returns the per-step global losses (device)."""
        if losses is None:
            pre = getattr(self, "_losses", None)
            losses = pre if (self.comm == "p2p" and pre is not None and pre.numel() >= n_steps) else \
                torch.empty(max(1, n_steps), dtype=torch.float64, device=self.dev)
        if self.comm == "p2p":
            bad = C.c_int64(-1)
            per_rank = max(1, self.batch_global // self.world)
            rc = L.lib().drb_mf_bpr_train_steps_p2p(_ptr(self.P), _ptr(self.ws.buf), max(1, self.U_local), self.I, self.F,
                                                    self._peer_ptrs, self.rank, self.world, _ptr(self.bu), _ptr(self.bi),
                                                    _ptr(self.bj), _ptr(self.step_offsets), int(self.offsets_host[-1]),
                                                    per_rank, first, n_steps, C.byref(self.hp), self.opt_steps, _ptr(losses),
                                                    C.c_double(self.peer_timeout_s), 0, C.byref(bad), _stream())
            L.check(rc)
            self.opt_steps += n_steps
        elif self.comm == "nccl":
            offs = np.ascontiguousarray(self.offsets_host, np.int64)
            L.check(L.lib().drb_mf_bpr_train_steps_sharded(_ptr(self.P), _ptr(self.Q), _ptr(self.ws.buf), max(1, self.U_local),
                                                           self.I, self.F, _ptr(self.bu), _ptr(self.bi), _ptr(self.bj),
                                                           offs.ctypes.data, first, n_steps, C.byref(self.hp), self.opt_steps,
                                                           _ptr(losses), _stream()))
            self.opt_steps += n_steps
        else:
            for k in range(n_steps):
                self.step(first + k)
                losses[k] = self.loss[0]
        return losses[:n_steps]

    def train_steps_host(self, h_bu, h_bi, h_bj, h_offsets, first, n_steps):
        """Global steps fed from pinned HOST planes holding this rank's share of every global batch (native loop: the
        H2D of step s+1 overlaps step s, one loss D2H per step).  Returns the per-step GLOBAL losses (pinned CPU fp64)."""
        if self.comm == "p2p":
            return self._train_steps_host_p2p(h_bu, h_bi, h_bj, h_offsets, first, n_steps)
        if self.comm != "nccl":
            raise RuntimeError("train_steps_host needs the native NCCL communicator or the peer kernel")
        offs = np.ascontiguousarray(h_offsets, np.int64)
        widest = int(np.diff(offs[first:first + n_steps + 1]).max()) if n_steps > 0 else 0
        stride = max(4, (widest + 3) // 4 * 4)
        if self._stage is None or self._stage.numel() < 6 * stride:
            self._stage = torch.empty(6 * stride, dtype=torch.int32, device=self.dev)
        d_loss = torch.empty(max(1, n_steps), dtype=torch.float64, device=self.dev)
        h_loss = torch.empty(max(1, n_steps), dtype=torch.float64).pin_memory()
        L.check(L.lib().drb_mf_bpr_train_steps_sharded_host(
            _ptr(self.P), _ptr(self.Q), _ptr(self.ws.buf), max(1, self.U_local), self.I, self.F, h_bu.data_ptr(),
            h_bi.data_ptr(), h_bj.data_ptr(), offs.ctypes.data, first, n_steps, C.byref(self.hp), self.opt_steps,
            _ptr(self._stage), stride, _ptr(d_loss), h_loss.data_ptr(), _stream()))
        self.opt_steps += n_steps
        return h_loss[:n_steps]

    def _train_steps_host_p2p(self, h_bu, h_bi, h_bj, h_offsets, first, n_steps, chunk=8):
        """Peer-kernel form: the host shares are copied in chunks of `chunk` global steps (side stream) under the persistent
        launch of the chunk before; the losses of a chunk come back with one D2H."""
        offs = np.ascontiguousarray(h_offsets, np.int64)
        assert np.array_equal(offs, self.offsets_host[:len(offs)]), "host shares must follow the prepared epoch's offsets"
        main = torch.cuda.current_stream(self.dev)
        if getattr(self, "_copy_stream", None) is None:
            self._copy_stream = torch.cuda.Stream(self.dev)
        # loss buffers live with the trainer: no device / pinned allocation while peers may already sit in their launch
        if getattr(self, "_loss_bufs", None) is None or self._loss_bufs[0].numel() < max(1, n_steps):
            self._loss_bufs = (torch.empty(max(64, n_steps), dtype=torch.float64, device=self.dev),
                               torch.empty(max(64, n_steps), dtype=torch.float64).pin_memory())
        d_loss, h_loss = self._loss_bufs
        self._copy_stream.wait_stream(main)
        spans = [(s, min(chunk, first + n_steps - s)) for s in range(first, first + n_steps, chunk)]
        ready = []
        for s0, k in spans:                                          # enqueue every copy; each chunk's launch waits for its own
            b, e = int(offs[s0]), int(offs[s0 + k])
            with torch.cuda.stream(self._copy_stream):
                for dst, src in ((self.bu, h_bu), (self.bi, h_bi), (self.bj, h_bj)):
                    dst[b:e].copy_(src[b:e], non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(self._copy_stream)
            ready.append(ev)
        for (s0, k), ev in zip(spans, ready):
            main.wait_event(ev)
            self.train_steps(s0, k, d_loss[s0 - first:])
            h_loss[s0 - first:s0 - first + k].copy_(d_loss[s0 - first:s0 - first + k], non_blocking=True)
        main.synchronize()
        return h_loss[:n_steps].clone()

    def step_host(self, h_bu, h_bi, h_bj, stage):
        """End-to-end step from pinned HOST arrays holding this rank's share of the global batch."""
        n = len(h_bu)
        stride = (n + 3) // 4 * 4
        for k, h in enumerate((h_bu, h_bi, h_bj)):
            stage[k * stride:k * stride + n].copy_(h if isinstance(h, torch.Tensor) else torch.from_numpy(h), non_blocking=True)
        self.step_device(stage[0:], stage[stride:], stage[2 * stride:], 0, n)
        return float(self.loss.item())                           # D2H of the global loss

    def check_nan(self):
        hdr = self.ws.buf[:256].cpu().numpy()
        status = int(np.frombuffer(hdr[144:148].tobytes(), np.int32)[0])   # WsHeader: barrier 8 + acc 128 + nan_step 8
        if status == L.DRB_ERR_NAN_LOSS:
            raise ValueError(L.NAN_LOSS_MESSAGE)
        if status == L.DRB_ERR_PEER:
            raise RuntimeError("multi-GPU peer exchange timed out: a rank did not reach the rendezvous (see DESIGN.md, "
                               "multi-GPU section); the NCCL step (sharded_comm='nccl') is the fallback")
