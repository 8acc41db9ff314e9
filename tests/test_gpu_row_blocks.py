"""The row-blocked path of the single-GPU provers (pb_prove_chips / pb_prove_segment with a memory budget below the resident footprint,
include/powdr_b200.h): the chips of the tallest heights keep their coefficients and one row block of each LDE, every phase recomputes
the blocks it reads, and the proof is the resident proof word for word.  B is forced with a budget from pb_footprint_bytes."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_chips import _chips
from util import P

pytestmark = pytest.mark.gpu


def _airs(ctx, chips):
    return [ctx.air(bc, spans, t.shape[0], bus) for t, bc, spans, bus in chips]


def _prove(ctx, airs, bufs, chips):
    arg = [(a, b.ptr, t.shape[1].bit_length() - 1, t.shape[0]) for a, b, (t, _, _, _) in zip(airs, bufs, chips)]
    return ctx.prove_chips(arg)


def _budget_for(airs, chips, lb):
    from powdr_b200.capi import footprint_bytes
    return footprint_bytes([(t.shape[1].bit_length() - 1, t.shape[0], a.perm_width) for a, (t, _, _, _) in zip(airs, chips)], lb)


def _check_stage_clocks(ctx):
    ms = ctx.last_stage_ms()
    parts = sum(v for k, v in ms.items() if k != "total")
    assert abs(parts - ms["total"]) <= 1e-3 * ms["total"] + 0.05, ms


@pytest.mark.parametrize("spec,lbs", [
    # heights 2^8 (two chips, one without interactions), 2^5 and 2^3: at B = 16 only 2^8 is blocked, at B = 4 also 2^5
    ([(8, 12, 0, 7), (8, 9, 2, 0), (5, 14, 0, 5), (3, 10, 0, 3)], [1, 2, 3, 4]),
    ([(7, 12, 4, 5), (3, 8, 3, 0), (7, 6, 2, 2)], [1, 3]),          # with AIR constraints
    ([(7, 9, 3, 0), (6, 5, 2, 0)], [2, 3]),                          # no interactions anywhere
    ([(4, 10, 0, 3), (9, 8, 2, 0)], [2, 3]),                         # the tallest chip is not the first and has no interactions
])
def test_blocked_chips_equal_the_resident_proof_and_the_oracle(ctx, orc, spec, lbs):
    chips = _chips(spec, seed=len(spec) + 40)
    airs = _airs(ctx, chips)
    bufs = [ctx.to_device(t) for t, _, _, _ in chips]
    try:
        ctx.set_memory_budget(0)
        resident = _prove(ctx, airs, bufs, chips)
        assert ctx.last_row_blocks() == 0
        e_proof, e_cs, e_ys, e_q = orc.prove_chips(chips, n_queries=8, pow_bits=4)
        assert resident[0] == e_proof
        for lb in lbs:
            ctx.set_memory_budget(_budget_for(airs, chips, lb))
            proof, cs, ys, q = _prove(ctx, airs, bufs, chips)
            assert ctx.last_row_blocks() == lb
            assert proof == e_proof, lb
            assert (cs == e_cs).all() and (ys == e_ys).all() and (q == e_q).all(), lb
            assert orc.verify_chips(chips, proof, cs, ys, q, check_constraints=False) == 0
            _check_stage_clocks(ctx)
    finally:
        ctx.set_memory_budget(0)
        for a in airs:
            a.free()


@pytest.mark.parametrize("on_device", [True, False])
def test_blocked_segment_equals_the_resident_segment(ctx, orc, on_device):
    chips = _chips([(9, 11, 4, 6)], seed=41)
    trace, bc, spans, bus = chips[0]
    air = ctx.air(bc, spans, trace.shape[0], bus)
    d = ctx.to_device(trace)
    host = None
    try:
        if not on_device:                     # a host-resident trace: pinned Montgomery words
            mont = ((trace.astype(np.uint64) * ((1 << 32) % P)) % P).astype(np.uint32)
            host = ctx.host_alloc(mont.nbytes)
            C.memmove(host, mont.ctypes.data, mont.nbytes)
        src = d.ptr if on_device else host
        ctx.set_memory_budget(0)
        ref = ctx.prove_segment(air, src, 9, trace.shape[0], on_device=on_device)
        ref_q, ref_ys = ctx.query_segment(9, trace.shape[0], air.perm_width)
        extra = 0 if on_device else trace.nbytes          # the copy of a host-resident trace counts
        for lb in (2, 4):
            ctx.set_memory_budget(_budget_for([air], chips, lb) + extra)
            proof = ctx.prove_segment(air, src, 9, trace.shape[0], on_device=on_device)
            assert ctx.last_row_blocks() == lb
            q, ys = ctx.query_segment(9, trace.shape[0], air.perm_width)
            assert proof == ref and (q == ref_q).all() and (ys == ref_ys).all(), lb
            _check_stage_clocks(ctx)
        e_proof, e_cs, e_ys, e_q = orc.prove_chips(chips, n_queries=8, pow_bits=4)
        assert proof["cumulative_sum"] == e_cs[0].tolist() and (ys == e_ys).all() and (q == e_q).all()
    finally:
        ctx.set_memory_budget(0)
        if host:
            ctx.host_free(host)
        air.free()


def test_a_budget_below_every_footprint_fails_before_launching_and_drops_the_query_state(ctx):
    chips = _chips([(8, 12, 0, 7), (5, 9, 2, 0)], seed=42)
    airs = _airs(ctx, chips)
    bufs = [ctx.to_device(t) for t, _, _, _ in chips]
    from powdr_b200.capi import Chip, ChipsProof
    arr = (Chip * 2)(*[Chip(a.h.value, b.ptr, t.shape[1].bit_length() - 1, t.shape[0]) for a, b, (t, _, _, _) in zip(airs, bufs, chips)])
    try:
        _prove(ctx, airs, bufs, chips)                                   # a queryable proof
        ctx.set_memory_budget(min(_budget_for(airs, chips, lb) for lb in range(5)) - 1)
        launches = ctx.launch_count()
        proof, cs = ChipsProof(), np.zeros((2, 4), dtype=np.uint32)
        assert ctx.lib.pb_prove_chips(ctx.h, arr, C.c_size_t(2), C.byref(proof), cs.ctypes.data_as(C.c_void_p)) == 2
        assert ctx.launch_count() == launches
        assert ctx.lib.pb_query_chips(ctx.h, None, C.c_size_t(0), None, C.c_size_t(0)) == -1
        ctx.set_memory_budget(0)
        _prove(ctx, airs, bufs, chips)
        assert ctx.last_row_blocks() == 0
    finally:
        ctx.set_memory_budget(0)
        for a in airs:
            a.free()


def test_keccak_logup_shape_at_2p21_rows_beyond_hbm(ctx, orc):
    """2^21 x 2022 with the 1734-interaction AIR of test_gpu_fullsize: about 113 GiB of resident matrices beside a 17 GB trace, proved
    on one H100 in row blocks; checked by the independent verifier, which includes the LogUp identity at zeta"""
    import torch
    from powdr_b200 import machine as M
    log_n, width = 21, 2022
    mach = M.SymbolicMachine([], M.synthetic_bus(width, 1734, seed=0xB2000002))
    w = mach.width
    bus = M.compile_bus(mach, 1)
    air = ctx.air([], [], w, bus)
    gen = torch.Generator(device="cuda").manual_seed(0xB2000021)
    trace = torch.randint(0, P, (w, 1 << log_n), dtype=torch.int32, device="cuda", generator=gen)
    try:
        assert ctx.lib.pb_to_monty(ctx.h, C.c_void_p(trace.data_ptr()), C.c_size_t(trace.numel())) == 0
        torch.cuda.synchronize()
        from powdr_b200.capi import footprint_bytes
        ctx.set_memory_budget(footprint_bytes([(log_n, w, air.perm_width)], 3))
        proof = ctx.prove_segment(air, trace.data_ptr(), log_n, w, on_device=True)
        assert ctx.last_row_blocks() >= 3
        queries, ys = ctx.query_segment(log_n, w, air.perm_width)
    finally:
        ctx.set_memory_budget(0)
        del trace
        torch.cuda.empty_cache()
    assert proof["final_poly"][0] == proof["final_poly"][1]
    assert orc.verify_segment([], [], log_n, w, proof, ys, queries, check_constraints=True, bus=bus) == 0
    air.free()
