"""Multi-GPU layout of the packing environments: bins are independent, so they are partitioned
contiguously by env index, one process per GPU, with NO collective inside a step.  The only exchange
is the end-of-rollout gather of observations / masks to every learner rank (SURVEY.md 8e); the
reference has no counterpart (single host, pipes: wrapper/shmem_vec_env.py:47-57).

Works with any ``torch.distributed`` backend (``nccl`` on GPUs, ``gloo`` in the CPU tests)."""
import numpy as np


def shard_range(num_envs_total, rank, world_size):
    """Contiguous block [lo, hi) of env indices owned by ``rank`` (sizes differ by at most one)."""
    base, rem = divmod(num_envs_total, world_size)
    lo = rank * base + min(rank, rem)
    hi = lo + base + (1 if rank < rem else 0)
    return lo, hi


def shard_sequences(sequences, rank, world_size):
    lo, hi = shard_range(len(sequences), rank, world_size)
    return np.ascontiguousarray(sequences[lo:hi])


def candidate_mask(obs, selected_action):
    """The action mask is column 4 of the candidate rows (reference tools.py:298-299)."""
    n = obs.shape[0]
    return obs[:, :selected_action * 5].reshape(n, selected_action, 5)[:, :, 4]


def gather_rollout(local, world_size=None, group=None):
    """All-gather a per-rank tensor ``[n_local, ...]`` (equal n_local on every rank) into
    ``[world * n_local, ...]`` ordered by rank, i.e. by global env index."""
    import torch
    import torch.distributed as dist
    if world_size is None:
        world_size = dist.get_world_size(group)
    if world_size == 1:
        return local
    local = local.contiguous()
    out = torch.empty((world_size * local.shape[0],) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out, local, group=group)
    return out


class _Works(object):
    def __init__(self, works):
        self.works = works

    def wait(self):
        for w in self.works:
            w.wait()


class AsyncRolloutGather(object):
    """The rollout-end gather taken off the critical path (SURVEY.md 8e: "overlap with the next step's
    scan"): ``start(local)`` enqueues the all-gather of a finished rollout's tensor on a side stream
    (after everything already enqueued on the caller's current stream), the caller goes on stepping the
    next rollout, ``finish()`` makes the current stream wait for the gather and returns the gathered
    tensor.  Two output buffers alternate, so a gathered tensor stays valid while the next gather is in
    flight.  On CPU tensors (gloo, the tests) the collective simply runs asynchronously."""

    def __init__(self, world_size=None, group=None, point_to_point=False):
        import torch.distributed as dist
        self.world = dist.get_world_size(group) if world_size is None else world_size
        self.group = group
        self.point_to_point = point_to_point    # the gather as world-1 send/recv pairs (NCCL can serve those with the
        if point_to_point:                      # copy engines, NCCL_P2P_USE_CUDA_MEMCPY=1) instead of the all-gather kernel
            self.kind = "nccl send/recv pairs"
        self._bufs = [None, None]
        self._turn = 0
        self._work = None
        self._out = None
        self._side = None
        self.events = None                      # (start, end) CUDA events of the last gather on the side stream

    def start(self, local):
        import torch
        import torch.distributed as dist
        if self._work is not None:
            raise RuntimeError("a gather is already in flight")
        local = local.contiguous()
        if self.world == 1:
            self._out, self._work = local, False
            return
        shape = (self.world * local.shape[0],) + tuple(local.shape[1:])
        buf = self._bufs[self._turn]
        if buf is None or buf.shape != shape or buf.dtype != local.dtype or buf.device != local.device:
            buf = torch.empty(shape, dtype=local.dtype, device=local.device)
            self._bufs[self._turn] = buf
        self._turn ^= 1
        if local.is_cuda:
            if self._side is None:
                self._side = torch.cuda.Stream(device=local.device)
            cur = torch.cuda.current_stream(local.device)
            self._side.wait_stream(cur)                       # `local` is complete in stream order
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.cuda.stream(self._side):
                e0.record()
                if self.point_to_point:
                    for w in self._pairs(buf, local):
                        w.wait()                              # stream-ordered for NCCL: the side stream waits, not the host
                else:
                    dist.all_gather_into_tensor(buf, local, group=self.group)
                e1.record()
            local.record_stream(self._side)
            self.events = (e0, e1)
            self._work = True
        elif self.point_to_point:
            self._work = _Works(self._pairs(buf, local))
        else:
            self._work = dist.all_gather_into_tensor(buf, local, group=self.group, async_op=True)
        self._out = buf

    def _pairs(self, buf, local):
        import torch.distributed as dist
        me, n = dist.get_rank(self.group), local.shape[0]
        buf[me * n:(me + 1) * n].copy_(local, non_blocking=True)
        ops = []
        for d in range(1, self.world):
            to, frm = (me + d) % self.world, (me - d) % self.world
            ops.append(dist.P2POp(dist.isend, local, to, self.group))
            ops.append(dist.P2POp(dist.irecv, buf[frm * n:(frm + 1) * n], frm, self.group))
        return dist.batch_isend_irecv(ops)

    def finish(self):
        import torch
        if self._work is None:
            raise RuntimeError("no gather in flight")
        if self._work is True:
            torch.cuda.current_stream(self._out.device).wait_stream(self._side)
        elif self._work is not False:
            self._work.wait()
        out, self._out, self._work = self._out, None, None
        return out


class CompactRolloutGather(object):
    """AsyncRolloutGather over the compact form of the location observation (``csrc/irbpp_pack.cuh``: 7 184 instead of
    14 132 bytes per bin at selectedAction = 500, lossless): pack on the sender, all-gather the packed rows, expand on the
    receiver.  The gather's duration -- and with it the stretch of steps it disturbs -- halves, at the cost of the two
    extra kernels.  CUDA tensors only (the kernels are in libirbpp)."""

    def __init__(self, selected_action, world_size=None, group=None):
        import ctypes
        from . import _lib
        self._lib = _lib.load()
        self._ct = ctypes
        self.sel = int(selected_action)
        self.row_bytes = int(self._lib.irbpp_packed_obs_bytes(self.sel))
        self._inner = AsyncRolloutGather(world_size, group)
        self.world = self._inner.world
        self._full = [None, None]
        self._turn = 0
        self._pending = None
        self.kind = "nccl all-gather of packed observations (%d of %d bytes per bin)" % (self.row_bytes, (self.sel * 5 + 9 + 1024) * 4)

    @property
    def events(self):
        return self._inner.events

    def start(self, local):
        import torch
        n = local.shape[0]
        packed = torch.empty((n, self.row_bytes), dtype=torch.uint8, device=local.device)
        st = torch.cuda.current_stream(local.device).cuda_stream
        p0, p1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        p0.record()
        rc = self._lib.irbpp_pack_observations(local.data_ptr(), local.stride(0), self.sel, n, packed.data_ptr(), st)
        p1.record()
        self.pack_events = (p0, p1)                          # the pack and the expansion run on the caller's stream
        if rc != 0:
            raise RuntimeError("irbpp_pack_observations failed: %s" % self._lib.irbpp_last_error(None))
        self._inner.start(packed)
        self._pending = (n, local.shape[1], local.device)

    def finish(self):
        import torch
        n, width, dev = self._pending
        gathered = self._inner.finish()                      # [world * n, row_bytes] uint8, current stream waits for it
        t = self._turn
        self._turn ^= 1
        full = self._full[t]
        if full is None or full.shape != (self.world * n, width):
            full = self._full[t] = torch.empty((self.world * n, width), dtype=torch.float32, device=dev)
        st = torch.cuda.current_stream(dev).cuda_stream
        u0, u1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        u0.record()
        rc = self._lib.irbpp_unpack_observations(gathered.data_ptr(), self.sel, self.world * n, full.data_ptr(), full.stride(0), st)
        u1.record()
        self.unpack_events = (u0, u1)
        if rc != 0:
            raise RuntimeError("irbpp_unpack_observations failed: %s" % self._lib.irbpp_last_error(None))
        self._pending = None
        return full


class PeerCopyGather(object):
    """The rollout gather as peer-to-peer copies by the COPY ENGINES instead of an NCCL kernel: every rank pushes its
    shard straight into every peer's gathered buffer over NVLink (the buffers are exchanged once as CUDA IPC handles),
    then a 4-byte NCCL all-reduce on the same side stream tells each rank that all pushes into ITS buffer are done.
    An NCCL all-gather occupies SMs on every GPU for its whole duration, and beside the latency-bound step kernels
    it cost almost as much step time as it took itself;
    copy-engine traffic does not compete for SMs, so it really runs beside the next rollout's steps.
    Same interface as AsyncRolloutGather; a gathered buffer stays valid until the second next ``start``.
    One node only (CUDA IPC); falls back to AsyncRolloutGather if the handles cannot be exchanged."""

    def __init__(self, world_size=None, group=None):
        import torch.distributed as dist
        self.world = dist.get_world_size(group) if world_size is None else world_size
        self.rank = dist.get_rank(group)
        self.group = group
        self._views = None            # [turn][peer rank] -> that peer's gathered buffer (own buffer for peer == rank)
        self._turn = 0
        self._side = None
        self._inflight = None
        self._fallback = None
        self.events = None
        self.kind = "peer-copy (copy engines over NVLink + 4-byte all-reduce)"

    def _setup(self, local):
        import torch
        import torch.distributed as dist
        from torch.multiprocessing.reductions import rebuild_cuda_tensor, reduce_tensor
        shape = (self.world * local.shape[0],) + tuple(local.shape[1:])
        own = [torch.empty(shape, dtype=local.dtype, device=local.device) for _ in range(2)]
        mine = [reduce_tensor(b)[1] for b in own]                  # CUDA IPC handles of both buffers
        everyone = [None] * self.world
        dist.all_gather_object(everyone, mine, group=self.group)
        self._views = [[own[t] if r == self.rank else rebuild_cuda_tensor(*everyone[r][t]) for r in range(self.world)]
                       for t in range(2)]
        self._token = torch.zeros(1, dtype=torch.int32, device=local.device)
        self._side = torch.cuda.Stream(device=local.device)
        self._n = local.shape[0]

    def start(self, local):
        import torch
        import torch.distributed as dist
        if self._inflight is not None:
            raise RuntimeError("a gather is already in flight")
        local = local.contiguous()
        if self._fallback is None and self._views is None:
            try:
                self._setup(local)
            except Exception as exc:                                # no IPC (other node, containers without it, ...)
                self._fallback = AsyncRolloutGather(self.world, self.group)
                self.kind = "nccl all-gather (peer-copy set-up failed: %s)" % type(exc).__name__
        if self._fallback is not None:
            self._fallback.start(local)
            self._inflight = "fallback"
            return
        t = self._turn
        self._turn ^= 1
        cur = torch.cuda.current_stream(local.device)
        self._side.wait_stream(cur)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        lo = self.rank * self._n
        with torch.cuda.stream(self._side):
            e0.record()
            for k in range(self.world):                             # start with the next rank: spreads the traffic over the links
                r = (self.rank + 1 + k) % self.world
                self._views[t][r][lo:lo + self._n].copy_(local, non_blocking=True)
            dist.all_reduce(self._token, group=self.group)          # completes when every rank has issued its pushes behind it
            e1.record()
        local.record_stream(self._side)
        self.events = (e0, e1)
        self._inflight = self._views[t][self.rank]

    def finish(self):
        import torch
        if self._inflight is None:
            raise RuntimeError("no gather in flight")
        if self._inflight == "fallback":
            out = self._fallback.finish()
            self.events = self._fallback.events
        else:
            out = self._inflight
            torch.cuda.current_stream(out.device).wait_stream(self._side)
        self._inflight = None
        return out


class SymmMemGather(object):
    """The rollout gather by the COPY ENGINES over torch's symmetric memory (``torch.distributed._symmetric_memory``:
    cuMem allocations mapped into every rank of the node): each rank publishes its shard in a symmetric buffer, a
    barrier, every rank PULLS the other shards straight into its gathered tensor with device-to-device copies over
    NVLink, a second barrier releases the buffers.  No SM runs the transfer (the barriers are one-CTA kernels), so
    unlike an NCCL all-gather kernel it does not take SM slots from the latency-bound step kernels beside it.
    Same interface as AsyncRolloutGather; falls back to it when symmetric memory cannot be set up (other node,
    no peer access)."""

    def __init__(self, world_size=None, group=None):
        import torch.distributed as dist
        self.world = dist.get_world_size(group) if world_size is None else world_size
        self.group = group
        self.rank = dist.get_rank(group)
        self._hdl = None
        self._src = None
        self._bufs = [None, None]
        self._turn = 0
        self._side = None
        self._out = None
        self._fallback = None
        self.events = None
        self.kind = "symmetric-memory pull (copy engines over NVLink)"

    def _setup(self, local):
        import torch
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm_mem
        group = self.group if self.group is not None else dist.group.WORLD
        self._src = symm_mem.empty(tuple(local.shape), dtype=local.dtype, device=local.device)
        self._hdl = symm_mem.rendezvous(self._src, group)
        # high priority: the two one-CTA barrier kernels must not queue behind a step kernel whose grid fills every SM slot
        self._side = torch.cuda.Stream(device=local.device, priority=-1)
        self._shape, self._dtype = tuple(local.shape), local.dtype

    def start(self, local):
        import torch
        if self._out is not None:
            raise RuntimeError("a gather is already in flight")
        local = local.contiguous()
        if self._fallback is None and self._hdl is None:
            try:
                self._setup(local)
            except Exception as exc:
                self._fallback = AsyncRolloutGather(self.world, self.group)
                self.kind = "nccl all-gather (symmetric memory set-up failed: %s: %s)" % (type(exc).__name__, str(exc)[:120])
        if self._fallback is not None:
            self._fallback.start(local)
            self._out = "fallback"
            return
        if tuple(local.shape) != self._shape or local.dtype != self._dtype:
            raise ValueError("the gathered tensor must keep its shape and dtype")
        n = local.shape[0]
        t = self._turn
        self._turn ^= 1
        buf = self._bufs[t]
        if buf is None:
            buf = self._bufs[t] = torch.empty((self.world * n,) + self._shape[1:], dtype=self._dtype, device=local.device)
        cur = torch.cuda.current_stream(local.device)
        self._side.wait_stream(cur)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(self._side):
            e0.record()
            self._src.copy_(local, non_blocking=True)                # publish
            self._hdl.barrier()                                      # every shard is published
            buf[self.rank * n:(self.rank + 1) * n].copy_(local, non_blocking=True)
            for step in range(1, self.world):                        # rank r starts at r - 1: no two ranks pull from one peer at once
                r = (self.rank - step) % self.world
                buf[r * n:(r + 1) * n].copy_(self._hdl.get_buffer(r, self._shape, self._dtype), non_blocking=True)
            self._hdl.barrier()                                      # every rank is done reading: the buffers may be rewritten
            e1.record()
        local.record_stream(self._side)
        self.events = (e0, e1)
        self._out = buf

    def finish(self):
        import torch
        if self._out is None:
            raise RuntimeError("no gather in flight")
        if isinstance(self._out, str):
            out = self._fallback.finish()
            self.events = self._fallback.events
        else:
            out = self._out
            torch.cuda.current_stream(out.device).wait_stream(self._side)
        self._out = None
        return out


def scatter_actions(global_actions, rank, world_size):
    """Slice of a global action vector (ordered by global env index) that belongs to ``rank``."""
    lo, hi = shard_range(global_actions.shape[0], rank, world_size)
    return global_actions[lo:hi]
