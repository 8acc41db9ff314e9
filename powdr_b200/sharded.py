"""Collectives for pb_prove_segment_sharded and pb_prove_chips_sharded (include/powdr_b200.h, pb_comm_t): the library takes two callbacks on DEVICE
pointers and links no communication library itself.

  TorchComm   -- one process per GPU, torch.distributed (NCCL over NVLink/NVSwitch); what bench.py uses for --gpus N > 1
  ThreadComm  -- G threads of one process on ONE GPU, a barrier plus host staging; the single-GPU parity harness
                 (tests/test_gpu_sharded.py): same library code path as NCCL, no second GPU needed

prove_chips_group runs the same provers without a pb_comm_t of ours: the library's group (pb_prove_chips_group) owns the rank threads
and exchanges device to device.
"""
import ctypes as C
import threading

import numpy as np

from .capi import load_library, _chk

COLLECTIVE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t)


class PbComm(C.Structure):
    _fields_ = [("rank", C.c_int), ("world", C.c_int), ("all_gather", COLLECTIVE_FN), ("all_to_all", COLLECTIVE_FN), ("user", C.c_void_p),
                ("flags", C.c_uint32)]


PB_COMM_STREAM_ORDERED = 1


def shard_columns(width, world, rank):
    """(first, count) of `rank`'s column block -- pb_shard_columns"""
    first, count = C.c_size_t(), C.c_size_t()
    _chk(load_library().pb_shard_columns(C.c_size_t(width), C.c_int(world), C.c_int(rank), C.byref(first), C.byref(count)), "pb_shard_columns")
    return first.value, count.value


class Comm:
    """Base: wraps two python callables (send_ptr, recv_ptr, nbytes) into a pb_comm_t; exceptions become PB_ERR_COMM."""

    def __init__(self, rank, world, flags=0):
        self.rank, self.world = rank, world
        self.error = None

        def wrap(fn):
            def cb(_user, send, recv, nbytes):
                try:
                    fn(int(send or 0), int(recv or 0), int(nbytes))
                    return 0
                except BaseException as e:      # noqa: BLE001 -- must not propagate into C
                    self.error = e
                    return 1
            return COLLECTIVE_FN(cb)

        self._ag, self._a2a = wrap(self.all_gather), wrap(self.all_to_all)      # keep the thunks alive
        self.c = PbComm(rank, world, self._ag, self._a2a, None, flags)

    def all_gather(self, send, recv, nbytes):
        raise NotImplementedError

    def all_to_all(self, send, recv, nbytes):
        raise NotImplementedError


class _DevBytes:
    """zero-copy view of raw device memory for torch.as_tensor"""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 3}


class TorchComm(Comm):
    """torch.distributed process group (backend nccl), one rank per GPU.  STREAM-ORDERED (PB_COMM_STREAM_ORDERED): the context must
    have been created on torch's current stream; a synchronous torch NCCL collective waits for the work already on that stream and
    makes the stream wait for the collective, so no host synchronisation is needed on either side."""

    def __init__(self, group=None, stream_ordered=True):
        import torch
        import torch.distributed as dist
        self.torch, self.dist, self.group = torch, dist, group
        self.stream_ordered = stream_ordered
        super().__init__(dist.get_rank(group), dist.get_world_size(group), PB_COMM_STREAM_ORDERED if stream_ordered else 0)
        self.calls, self.bytes = 0, 0

    def _t(self, ptr, nbytes):
        return self.torch.as_tensor(_DevBytes(ptr, nbytes), device="cuda")

    def all_gather(self, send, recv, nbytes):
        self.dist.all_gather_into_tensor(self._t(recv, nbytes * self.world), self._t(send, nbytes), group=self.group)
        if not self.stream_ordered:
            self.torch.cuda.synchronize()
        self.calls += 1
        self.bytes += nbytes * self.world

    def all_to_all(self, send, recv, nbytes):
        self.dist.all_to_all_single(self._t(recv, nbytes * self.world), self._t(send, nbytes * self.world), group=self.group)
        if not self.stream_ordered:
            self.torch.cuda.synchronize()
        self.calls += 1
        self.bytes += nbytes * self.world


class ThreadGroup:
    """shared state of `world` ThreadComm ranks"""

    def __init__(self, world):
        self.world = world
        self.barrier = threading.Barrier(world)
        self.slots = [None] * world


class ThreadComm(Comm):
    """calls / bytes: collectives made and bytes received by this rank, per kind ("all_gather", "all_to_all")"""

    def __init__(self, group, rank, ctx):
        self.group, self.ctx = group, ctx
        self.calls = {"all_gather": 0, "all_to_all": 0}
        self.bytes = {"all_gather": 0, "all_to_all": 0}
        super().__init__(rank, group.world)

    def _d2h(self, ptr, nbytes):
        host = np.empty(nbytes, dtype=np.uint8)
        _chk(self.ctx.lib.pb_copy_d2h(self.ctx.h, host.ctypes.data_as(C.c_void_p), C.c_void_p(ptr), C.c_size_t(nbytes)), "pb_copy_d2h")
        self.ctx.synchronize()
        return host

    def _h2d(self, ptr, host):
        host = np.ascontiguousarray(host)
        _chk(self.ctx.lib.pb_copy_h2d(self.ctx.h, C.c_void_p(ptr), host.ctypes.data_as(C.c_void_p), C.c_size_t(host.nbytes)), "pb_copy_h2d")
        self.ctx.synchronize()

    def all_gather(self, send, recv, nbytes):
        g = self.group
        self.calls["all_gather"] += 1
        self.bytes["all_gather"] += nbytes * self.world
        g.slots[self.rank] = self._d2h(send, nbytes)
        g.barrier.wait(timeout=120)
        self._h2d(recv, np.concatenate(g.slots))
        g.barrier.wait(timeout=120)

    def all_to_all(self, send, recv, nbytes):
        g = self.group
        self.calls["all_to_all"] += 1
        self.bytes["all_to_all"] += nbytes * self.world
        g.slots[self.rank] = self._d2h(send, nbytes * self.world)
        g.barrier.wait(timeout=120)
        self._h2d(recv, np.concatenate([g.slots[r][self.rank * nbytes:(self.rank + 1) * nbytes] for r in range(self.world)]))
        g.barrier.wait(timeout=120)


def _run_ranks(world, body):
    """body(rank, group) on `world` threads; the first real error is raised (a broken barrier only follows another rank's error)"""
    group = ThreadGroup(world)
    out, errs = [None] * world, [None] * world

    def run(rank):
        try:
            out[rank] = body(rank, group)
        except BaseException as e:      # noqa: BLE001
            errs[rank] = e
            group.barrier.abort()

    threads = [threading.Thread(target=run, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for e in errs:
        if e is not None and not isinstance(e, threading.BrokenBarrierError):
            raise e
    for e in errs:
        if e is not None:
            raise e
    return out


def prove_chips_threads(world, chips, device=0, fri_params=(8, 4), want_queries=True, stats=None, comm_factory=None, budget=0):
    """Prove all chips of a segment under one transcript with `world` thread-ranks on one GPU (pb_prove_chips_sharded).  chips:
    [(trace canonical (W, N) uint32, bytecode, spans, bus or None)]; each rank compiles its own AIRs and passes its column block of
    every chip.  -> per rank the tuple of Context.prove_chips (proof dict, cumulative sums, opened values, queries or None).
    stats (optional list of `world` slots): per rank {"calls", "bytes", "launches", "stage_ms"} of the proof and query phase.
    comm_factory(group, rank, ctx) (optional) makes the rank's Comm instead of a ThreadComm.
    budget: every rank's pb_ctx_set_memory_budget (0: resident); stats then also has "log_blocks", pb_last_row_blocks."""
    from .capi import Context

    def body(rank, group):
        ctx = Context(device)
        try:
            ctx.set_fri_params(*fri_params)
            ctx.set_memory_budget(budget)
            airs, bufs, args = [], [], []
            for trace, bc, spans, bus in chips:
                width, n = trace.shape
                air = ctx.air(bc, spans, width, bus)
                first, count = shard_columns(width, world, rank)
                buf = ctx.to_device(trace[first:first + count]) if count else None
                airs.append(air)
                bufs.append(buf)
                args.append((air, buf.ptr if buf else 0, n.bit_length() - 1, width))
            comm = comm_factory(group, rank, ctx) if comm_factory else ThreadComm(group, rank, ctx)
            l0 = ctx.launch_count()
            res = ctx.prove_chips_sharded(args, comm, want_queries=want_queries)
            if comm.error:
                raise comm.error
            if stats is not None:
                stats[rank] = {"calls": dict(getattr(comm, "calls", {})), "bytes": dict(getattr(comm, "bytes", {})),
                               "launches": ctx.launch_count() - l0, "stage_ms": ctx.last_stage_ms(), "log_blocks": ctx.last_row_blocks()}
            for a in airs:
                a.free()
            return res
        finally:
            ctx.close()

    return _run_ranks(world, body)


def prove_segment_threads(world, trace, bytecode, spans, device=0, on_device=True, fri_params=(8, 4), bus=None, want_queries=False,
                          stage_ms=None, stats=None, budget=0):
    """Prove one segment with `world` thread-ranks on one GPU (parity harness).  trace: canonical (W, N) uint32.
    -> list of per-rank proof dicts (all equal); with want_queries, list of (proof dict, query openings) per rank.
    stage_ms (optional list of `world` slots): each rank's Context.last_stage_ms() after its proof.
    stats (optional list of `world` slots): each rank's collective calls and bytes (ThreadComm.calls / .bytes), kernel launches and
    "log_blocks" (pb_last_row_blocks).  budget: every rank's pb_ctx_set_memory_budget (0: resident)."""
    from .capi import Context
    width, n = trace.shape
    log_n = n.bit_length() - 1

    def body(rank, group):
        ctx = Context(device)
        try:
            ctx.set_fri_params(*fri_params)
            ctx.set_memory_budget(budget)
            air = ctx.air(bytecode, spans, width, bus)
            first, count = shard_columns(width, world, rank)
            comm = ThreadComm(group, rank, ctx)
            if on_device:
                buf = ctx.to_device(trace[first:first + count]) if count else None
                ptr = buf.ptr if buf else 0
            else:
                host = np.ascontiguousarray(trace[first:first + count])
                host = ((host.astype(np.uint64) * np.uint64((1 << 32) % 2013265921)) % np.uint64(2013265921)).astype(np.uint32)
                ptr = host.ctypes.data if count else 0
            l0 = ctx.launch_count()
            res = ctx.prove_segment_sharded(air, ptr, log_n, width, comm, on_device=on_device)
            if stage_ms is not None:
                stage_ms[rank] = ctx.last_stage_ms()
            if want_queries:
                res = (res, ctx.query_segment_sharded(comm, log_n, width, air.perm_width))
            if stats is not None:
                stats[rank] = {"calls": dict(comm.calls), "bytes": dict(comm.bytes), "launches": ctx.launch_count() - l0,
                               "log_blocks": ctx.last_row_blocks()}
            if comm.error:
                raise comm.error
            return res
        finally:
            ctx.close()

    return _run_ranks(world, body)


def prove_chips_group(world, chips, devices=None, fri_params=(8, 4), want_queries=True, stats=None, budget=0):
    """prove_chips_threads through the library's group (pb_prove_chips_group): `world` contexts, rank r on devices[r] (default: all on
    device 0), each with its own AIRs and its column block of every chip; one call proves on all of them, the library running the rank
    threads and the device-to-device exchanges.  -> the list prove_chips_threads returns, one entry per rank: the group's answer, which the
    library has checked equal on every rank.  stats (optional list of `world` slots): per rank {"launches", "stage_ms", "log_blocks"}.
    budget: every rank's pb_ctx_set_memory_budget (0: resident)."""
    from .capi import Context, Group
    devices = list(devices) if devices is not None else [0] * world
    ctxs, airs, bufs, args, group = [], [], [], [], None
    try:
        for rank in range(world):
            ctx = Context(devices[rank])        # makes its device current: the AIRs and the column blocks below go there
            ctxs.append(ctx)
            ctx.set_fri_params(*fri_params)
            ctx.set_memory_budget(budget)
            mine = []
            for trace, bc, spans, bus in chips:
                width, n = trace.shape
                air = ctx.air(bc, spans, width, bus)
                first, count = shard_columns(width, world, rank)
                buf = ctx.to_device(trace[first:first + count]) if count else None
                airs.append(air)
                bufs.append(buf)
                mine.append((air, buf.ptr if buf else 0, n.bit_length() - 1, width))
            args.append(mine)
        group = Group(ctxs)
        l0 = [c.launch_count() for c in ctxs]
        res = group.prove_chips(args, want_queries=want_queries)
        if stats is not None:
            for r, c in enumerate(ctxs):
                stats[r] = {"launches": c.launch_count() - l0[r], "stage_ms": c.last_stage_ms(), "log_blocks": c.last_row_blocks()}
        return [res] * world
    finally:
        if group is not None:
            group.close()
        for a in airs:
            a.free()
        for b in bufs:
            if b is not None:
                b.free()
        for c in ctxs:
            c.close()
