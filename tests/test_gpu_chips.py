"""GPU parity of the multi-chip segment proof under ONE transcript (pb_prove_chips / pb_query_chips, include/powdr_b200.h) against
the CPU restatement (oracle/prove.c orc_prove_chips) and its independent verifier (oracle/verify.c orc_verify_chips): mixed-height
MMCS commitments, shared challenges, per-height injection of the reduced openings into one FRI instance.
Reference shape: one proving context with an AirProvingContext per chip of the segment
(/root/reference/openvm/src/powdr_extension/trace_generator/cuda/mod.rs:415-419, /root/reference/openvm-riscv/src/lib.rs:327-332)."""
import numpy as np
import pytest

from util import rand_field

pytestmark = pytest.mark.gpu


def _chips(spec, seed=0, zero=False):
    """spec: list of (log_n, width, n_constraints, n_interactions[, zero trace]) -> [(trace, bytecode, spans, bus)]"""
    from powdr_b200 import machine as M
    rng = np.random.default_rng(seed)
    out = []
    for i, (log_n, width, ncons, nints, *z) in enumerate(spec):
        base = M.synthetic_machine(width, ncons, seed=100 + i) if ncons else None
        bus_json = M.synthetic_bus(width, nints, seed=200 + i, quadratic_every=5) if nints else []
        mach = M.SymbolicMachine(base.constraints if base else [], bus_json)
        bc, spans = M.compile_constraints(mach)
        bus = M.compile_bus(mach, 1) if nints else None
        trace = np.zeros((mach.width, 1 << log_n), dtype=np.uint32) if zero or (z and z[0]) else rand_field(rng, (mach.width, 1 << log_n))
        out.append((trace, bc, spans, bus))
    return out


def _gpu_prove(ctx, chips):
    airs = [ctx.air(bc, spans, t.shape[0], bus) for t, bc, spans, bus in chips]
    bufs = [ctx.to_device(t) for t, _, _, _ in chips]
    arg = [(a, b.ptr, t.shape[1].bit_length() - 1, t.shape[0]) for a, b, (t, _, _, _) in zip(airs, bufs, chips)]
    out = ctx.prove_chips(arg)
    for a in airs:
        a.free()
    return out


@pytest.mark.parametrize("spec", [
    [(6, 12, 0, 7), (4, 9, 2, 0), (4, 14, 0, 5), (3, 10, 0, 3)],        # heights 2^6, 2^4 (x2, one without interactions), 2^3
    [(5, 12, 4, 5), (3, 8, 3, 0), (4, 6, 2, 2)],                        # with AIR constraints
    [(4, 9, 3, 0), (4, 5, 2, 0)],                                       # no interactions anywhere: no permutation commitment
    [(3, 10, 0, 3), (7, 8, 2, 0)],                                      # the tallest chip is not the first and has no interactions
    [(8, 6, 2, 4), (8, 7, 0, 3), (8, 5, 1, 0)],                         # equal heights: one leaf row over all matrices
    [(4, 6, 1, 2), (4, 5, 0, 3), (4, 7, 2, 1), (4, 4, 1, 2), (4, 6, 0, 2)],   # 15 column runs at one height: a split reduced opening
])
def test_chips_proof_matches_oracle_bit_for_bit(ctx, orc, spec):
    chips = _chips(spec, seed=len(spec))
    proof, cs, ys, q = _gpu_prove(ctx, chips)
    e_proof, e_cs, e_ys, e_q = orc.prove_chips(chips, n_queries=8, pow_bits=4)
    assert proof["main_root"] == e_proof["main_root"]
    assert (cs == e_cs).all() and proof["perm_root"] == e_proof["perm_root"]
    assert proof["quotient_root"] == e_proof["quotient_root"]
    assert (ys == e_ys).all()
    assert proof["fri_roots"] == e_proof["fri_roots"]
    assert proof == e_proof and (q == e_q).all()
    assert orc.verify_chips(chips, proof, cs, ys, q, check_constraints=False) == 0


def test_one_chip_equals_the_single_chip_prover(ctx, orc):
    chips = _chips([(6, 11, 4, 6)], seed=2)
    proof, cs, ys, q = _gpu_prove(ctx, chips)
    trace, bc, spans, bus = chips[0]
    air = ctx.air(bc, spans, trace.shape[0], bus)
    d = ctx.to_device(trace)
    single = ctx.prove_segment(air, d.ptr, 6, trace.shape[0], on_device=True)
    q1, ys1 = ctx.query_segment(6, trace.shape[0], air.perm_width)
    assert proof["main_root"] == single["trace_root"] and proof["perm_root"] == single["perm_root"]
    assert proof["quotient_root"] == single["quotient_root"] and proof["fri_roots"] == single["fri_roots"]
    assert proof["pow_witness"] == single["pow_witness"] and (ys == ys1).all() and (q == q1).all()
    assert cs[0].tolist() == single["cumulative_sum"]
    shared = set(proof) & set(single)                   # every other field of the one-chip proof keeps its name
    assert len(shared) >= 14 and {k: proof[k] for k in shared} == {k: single[k] for k in shared}
    assert single["perm_width"] == air.perm_width


def test_satisfying_traces_verify_with_the_constraint_identity(ctx, orc):
    chips = _chips([(5, 12, 4, 5), (3, 8, 3, 0), (4, 6, 2, 2)], seed=3, zero=True)     # padding rows satisfy the guarded constraints
    proof, cs, ys, q = _gpu_prove(ctx, chips)
    assert orc.verify_chips(chips, proof, cs, ys, q, check_constraints=True) == 0
    rnd = _chips([(5, 12, 4, 5), (3, 8, 3, 0), (4, 6, 2, 2)], seed=3)
    proof, cs, ys, q = _gpu_prove(ctx, rnd)
    assert orc.verify_chips(rnd, proof, cs, ys, q, check_constraints=False) == 0
    assert orc.verify_chips(rnd, proof, cs, ys, q, check_constraints=True) == 16


def test_chips_at_scale_verify(ctx, orc):
    """2^14 / 2^12 / 2^9 rows with a few hundred interactions: beyond the scalar prover's reach in a test, so the check is the
    independent verifier (all challenges, three MMCS openings per query, every fold with its injection, the LogUp identities)"""
    chips = _chips([(14, 64, 0, 120), (12, 40, 0, 60), (9, 30, 3, 0, True), (12, 24, 0, 33)], seed=9)   # the constraint-only chip: padding rows
    proof, cs, ys, q = _gpu_prove(ctx, chips)
    assert proof["log_max"] == 15 and proof["final_poly"][0] == proof["final_poly"][1]
    assert orc.verify_chips(chips, proof, cs, ys, q, check_constraints=True) == 0
    # the whole state is replaced by the next proof: prove something smaller, then the same again
    small = _chips([(4, 9, 3, 0), (4, 5, 2, 0)], seed=2)
    p_small = _gpu_prove(ctx, small)
    assert orc.verify_chips(small, *p_small, check_constraints=False) == 0
    again = _gpu_prove(ctx, chips)
    assert again[0] == proof and (again[3] == q).all()


@pytest.mark.parametrize("first", ["chips", "segment", "failed_segment"])
def test_a_query_reads_only_the_proof_of_its_own_prover(ctx, first):
    """the context keeps one proof state: after a proof by another prover, or after a failed proof, a query is refused; a proof by the
    query's own prover makes it answer again"""
    import ctypes as C
    from powdr_b200.capi import SegmentProof
    lib = ctx.lib
    chips = _chips([(5, 12, 4, 5), (3, 8, 3, 0)], seed=4)
    trace, bc, spans, bus = chips[0]
    air = ctx.air(bc, spans, trace.shape[0], bus)
    d = ctx.to_device(trace)
    out = np.zeros(1 << 20, dtype=np.uint32)
    ptr, cap = out.ctypes.data_as(C.c_void_p), C.c_size_t(out.size)
    if first == "chips":
        _gpu_prove(ctx, chips)
        assert lib.pb_query_segment(ctx.h, ptr, cap) == -1
        assert lib.pb_last_openings(ctx.h, ptr, cap) == -1
    elif first == "segment":
        ctx.prove_segment(air, d.ptr, 5, trace.shape[0], on_device=True)
        assert lib.pb_query_chips(ctx.h, ptr, cap, None, C.c_size_t(0)) == -1
        _gpu_prove(ctx, chips)                          # queries its own proof (pb_query_chips) or raises
    else:
        ctx.prove_segment(air, d.ptr, 5, trace.shape[0], on_device=True)
        bad = lib.pb_prove_segment(ctx.h, air.h, C.c_void_p(d.ptr), C.c_size_t(5), C.c_size_t(trace.shape[0] + 1), C.c_uint32(1), C.byref(SegmentProof()))
        assert bad == -1
        assert lib.pb_query_segment(ctx.h, ptr, cap) == -1
    if first != "segment":
        ctx.prove_segment(air, d.ptr, 5, trace.shape[0], on_device=True)
        ctx.query_segment(5, trace.shape[0], air.perm_width)      # raises unless both the query and the opened values are returned
    air.free()


def test_argument_checks(ctx):
    import ctypes as C
    from powdr_b200.capi import Chip, ChipsProof
    lib = ctx.lib
    proof = ChipsProof()
    cs = (C.c_uint32 * 4)()
    arr = (Chip * 1)(Chip(None, None, 4, 3))
    assert lib.pb_prove_chips(ctx.h, arr, C.c_size_t(1), C.byref(proof), cs) == -1          # null air / trace
    assert lib.pb_prove_chips(ctx.h, arr, C.c_size_t(0), C.byref(proof), cs) == -1
    assert lib.pb_query_chips(ctx.h, None, C.c_size_t(0), None, C.c_size_t(0)) == -1          # nothing proved since the failure above

