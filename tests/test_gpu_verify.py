"""The library's host verifier (pb_verify_segment, pb_verify_chips) on proofs of the GPU provers: the single-chip prover with the
trace on the device and in host memory, chip mixes, the row-blocked path, the sharded provers at G = 2 and 4, and the headline shape
(2^20 x 2022, 1734 interactions, 100 queries, 16 proof-of-work bits).  A tampered query word is rejected with the oracle's code."""
import time

import numpy as np
import pytest

from test_gpu_chips import _chips, _gpu_prove
from util import P

pytestmark = pytest.mark.gpu

N_Q, POW = 8, 4          # the ctx fixture's FRI parameters


def _keys(chips):
    from powdr_b200 import VerifyingKey
    return [(VerifyingKey(bc, sp, t.shape[0], bus), t.shape[1].bit_length() - 1) for t, bc, sp, bus in chips]


def _accept_and_reject_tampered(orc, chips, proof, cs, ys, q, n_queries=N_Q, pow_bits=POW):
    from powdr_b200 import verify_chips
    from powdr_b200.capi import PB_ERR_REJECTED
    keys = _keys(chips)
    assert verify_chips(keys, proof, cs, ys, q, n_queries=n_queries, pow_bits=pow_bits) == (0, 0)
    q2 = q.copy()
    q2[1, 2] = (int(q2[1, 2]) + 1) % P                  # a word of the first chip's main row
    want = orc.verify_chips(chips, proof, cs, ys, q2, check_constraints=False)
    assert want == 8 and verify_chips(keys, proof, cs, ys, q2, n_queries=n_queries, pow_bits=pow_bits) == (PB_ERR_REJECTED, want)


@pytest.mark.parametrize("on_device", [True, False])
def test_segment_proofs_verify(ctx, orc, on_device):
    from powdr_b200 import verify_segment
    from powdr_b200.capi import PB_ERR_REJECTED
    (trace, bc, spans, bus), = _chips([(9, 14, 4, 6, True)], seed=5)
    air = ctx.air(bc, spans, trace.shape[0], bus)
    if on_device:
        d = ctx.to_device(trace)
        proof = ctx.prove_segment(air, d.ptr, 9, trace.shape[0], on_device=True)
    else:
        host = ((trace.astype(np.uint64) * np.uint64((1 << 32) % P)) % np.uint64(P)).astype(np.uint32)
        proof = ctx.prove_segment(air, host.ctypes.data, 9, trace.shape[0], on_device=False)
    q, ys = ctx.query_segment(9, trace.shape[0], air.perm_width)
    air.free()
    (vk, log_n), = _keys([(trace, bc, spans, bus)])
    assert verify_segment(vk, log_n, proof, ys, q, n_queries=N_Q, pow_bits=POW) == (0, 0)
    q2 = q.copy()
    q2[0, 5] = (int(q2[0, 5]) + 1) % P
    want = orc.verify_segment(bc, spans, 9, trace.shape[0], proof, ys, q2, bus=bus)
    assert want != 0 and verify_segment(vk, log_n, proof, ys, q2, n_queries=N_Q, pow_bits=POW) == (PB_ERR_REJECTED, want)


@pytest.mark.parametrize("spec", [
    [(6, 12, 0, 7), (4, 9, 2, 0, True), (4, 14, 0, 5), (3, 10, 0, 3)],
    [(5, 12, 4, 5, True), (3, 8, 3, 0, True), (4, 6, 2, 2, True)],
    [(1, 6, 0, 3), (2, 5, 2, 0, True), (7, 8, 0, 4)],
])
def test_chip_mixes_verify(ctx, orc, spec):
    chips = _chips(spec, seed=len(spec) + 60)
    _accept_and_reject_tampered(orc, chips, *_gpu_prove(ctx, chips))


def test_row_blocked_proofs_verify(ctx, orc):
    from powdr_b200.capi import footprint_bytes
    chips = _chips([(8, 12, 0, 7), (8, 9, 2, 0, True), (5, 14, 0, 5)], seed=70)
    airs = [ctx.air(bc, sp, t.shape[0], bus) for t, bc, sp, bus in chips]
    bufs = [ctx.to_device(t) for t, _, _, _ in chips]
    arg = [(a, b.ptr, t.shape[1].bit_length() - 1, t.shape[0]) for a, b, (t, _, _, _) in zip(airs, bufs, chips)]
    try:
        for lb in (1, 3):
            ctx.set_memory_budget(footprint_bytes([(t.shape[1].bit_length() - 1, t.shape[0], a.perm_width) for a, (t, _, _, _) in zip(airs, chips)], lb))
            out = ctx.prove_chips(arg)
            assert ctx.last_row_blocks() == lb
            _accept_and_reject_tampered(orc, chips, *out)
    finally:
        ctx.set_memory_budget(0)
        for a in airs:
            a.free()


@pytest.mark.parametrize("world", [2, 4])
def test_sharded_proofs_verify(orc, world):
    import ctypes as C
    from powdr_b200 import verify_segment
    from powdr_b200.capi import Context
    from powdr_b200.sharded import ThreadComm, _run_ranks, prove_chips_threads, shard_columns
    chips = _chips([(9, 10, 0, 5), (7, 9, 2, 0, True), (8, 12, 0, 4)], seed=world)
    for got in prove_chips_threads(world, chips):
        _accept_and_reject_tampered(orc, chips, *got)
    (trace, bc, spans, bus), = _chips([(9, 11, 3, 4, True)], seed=world + 1)
    (vk, log_n), = _keys([(trace, bc, spans, bus)])
    width = trace.shape[0]

    def body(rank, group):          # what an integrator of pb_prove_segment_sharded holds: proof, queries, pb_last_openings
        c = Context(0)
        try:
            c.set_fri_params(N_Q, POW)
            air = c.air(bc, spans, width, bus)
            first, count = shard_columns(width, world, rank)
            block = c.to_device(trace[first:first + count])
            comm = ThreadComm(group, rank, c)
            proof = c.prove_segment_sharded(air, block.ptr, log_n, width, comm, on_device=True)
            q = c.query_segment_sharded(comm, log_n, width, air.perm_width)
            ys = np.empty((width + 2 * air.perm_width + 8, 4), dtype=np.uint32)
            assert c.lib.pb_last_openings(c.h, ys.ctypes.data_as(C.c_void_p), C.c_size_t(ys.size)) == 0
            assert comm.error is None
            air.free()
            return proof, ys, q
        finally:
            c.close()

    for proof, ys, q in _run_ranks(world, body):
        assert verify_segment(vk, log_n, proof, ys, q, n_queries=N_Q, pow_bits=POW) == (0, 0)


def test_key_refusals_match_pb_air_compile(ctx):
    """pb_vk_create refuses bytecode exactly where pb_air_compile and pb_air_set_interactions do"""
    from powdr_b200.capi import PbError
    from test_verify_host import BAD_BUSES, BAD_CONSTRAINTS, _vk_rc
    import powdr_b200 as pb

    def air_rc(bc, spans, width, bus=None):
        try:
            ctx.air(bc, spans, width, bus).free()
            return 0
        except PbError as e:
            return e.code

    for bc, code in BAD_CONSTRAINTS:
        assert air_rc(bc, [(0, len(bc))], 3) == _vk_rc(pb, bc, [(0, len(bc))], 3) == code, bc
    for bus, code in BAD_BUSES:
        assert air_rc([], [], 4, bus) == _vk_rc(pb, [], [], 4, bus) == code, bus


def test_headline_shape_verifies(ctx):
    """2^20 x 2022 with the 1734-interaction AIR of test_gpu_fullsize.py at 100 queries and 16 proof-of-work bits: the GPU proof is
    accepted; the median host verification time of 5 runs is printed (DESIGN.md §3d)"""
    import ctypes as C
    from powdr_b200 import machine as M, verify_segment
    log_n, width = 20, 2022
    rng = np.random.default_rng(0xB2000001)
    mach = M.SymbolicMachine([], M.synthetic_bus(width, 1734, seed=0xB2000002))
    w = mach.width
    bus = M.compile_bus(mach, 1)
    trace = rng.integers(0, P, size=(w, 1 << log_n), dtype=np.uint32)
    air = ctx.air([], [], w, bus)
    d = ctx.alloc(trace.nbytes).upload(trace)
    assert ctx.lib.pb_to_monty(ctx.h, C.c_void_p(d.ptr), C.c_size_t(trace.size)) == 0
    del trace
    try:
        ctx.set_fri_params(100, 16)
        proof = ctx.prove_segment(air, d.ptr, log_n, w, on_device=True)
        q, ys = ctx.query_segment(log_n, w, air.perm_width)
    finally:
        ctx.set_fri_params(N_Q, POW)
        d.free()
        air.free()
    (vk, _), = _keys([(np.empty((w, 2), dtype=np.uint32), [], [], bus)])
    times = []
    for _ in range(5):
        t0 = time.perf_counter()
        assert verify_segment(vk, log_n, proof, ys, q, n_queries=100, pow_bits=16) == (0, 0)
        times.append(time.perf_counter() - t0)
    print("headline verification: median %.3f s, min %.3f s, max %.3f s over 5 runs on the host (%d queries, %d opened values, %d words per query)"
          % (float(np.median(times)), min(times), max(times), q.shape[0], ys.shape[0], q.shape[1]))
    q2 = q.copy()
    q2[99, q.shape[1] - 1] = (int(q2[99, q.shape[1] - 1]) + 1) % P       # the last FRI path word of the last query
    assert verify_segment(vk, log_n, proof, ys, q2, n_queries=100, pow_bits=16) == (-8, 12)
