"""The generated AIRs of tests/exprgen.py on the GPU, bit for bit against the plain evaluator (constraint fold, quotient) and the oracle
(whole proofs, periphery histograms):

  * ctx.constraint_fold and ctx.quotient through the NVRTC-generated kernels (air.is_jit asserted) and through the interpreter
    (PB_AIR_NO_JIT), on random and edge-valued matrices, at fold heights 1, 255, 257, 1000 and quotient heights 2^1, 2^2, 2^9, 2^12;
  * segment proofs with generated interactions, with and without generated constraints, and one multi-chip proof with a generated
    chip next to synthetic ones;
  * the refusals of ctx.air(..., bus) before any launch;
  * generated periphery interactions through both stage-0 kernels against orc.apc_apply_bus.

Seeds are fixed, so the on-disk JIT cache makes a second run cheap."""
import numpy as np
import pytest

import exprgen as G
from test_gpu_height_range import _check_chips, _check_segment
from test_gpu_chips import _chips
from test_gpu_tracegen import _bus_case
from util import P

pytestmark = pytest.mark.gpu

AIRS = {c.name: c for c in G.all_air_cases()}
BUSES = {c.name: c for c in G.bus_cases()}
ALPHA = [123456789, 987654321, 5, P - 1]


@pytest.mark.parametrize("mode", ["jit", "interpreter"])
@pytest.mark.parametrize("name", list(AIRS))
def test_fold_and_quotient_match_the_evaluator(ctx, name, mode, monkeypatch):
    case = AIRS[name]
    bc, spans = case.program()
    if mode == "interpreter":
        monkeypatch.setenv("PB_AIR_NO_JIT", "1")
    air = ctx.air(bc, spans, case.width)
    try:
        assert air.is_jit == (mode == "jit")
        for h in (1, 255, 257, 1000):
            for kind, mat in {"random": G.rand_matrix(case.width, h, h), "edge": G.edge_matrix(case.width, h, h)}.items():
                d = ctx.to_device(mat)
                out = ctx.alloc(16 * h)
                ctx.constraint_fold(air, d.ptr, h, ALPHA, out.ptr)
                assert (ctx.to_host(out, (4, h)) == case.fold(mat, ALPHA)).all(), (h, kind)
        for log_n in (1, 2, 9, 12):
            m = 2 << log_n
            for kind, lde in {"random": G.rand_matrix(case.width, m, log_n), "edge": G.edge_matrix(case.width, m, log_n)}.items():
                d = ctx.to_device(lde)
                q = ctx.alloc(4 * 8 << log_n)
                ctx.quotient(air, d.ptr, log_n, ALPHA, q.ptr)
                exp = G.quotient(case.fold(lde, ALPHA), log_n)
                assert (ctx.to_host(q, (2, 4, 1 << log_n)) == exp).all(), (log_n, kind)
    finally:
        air.free()


def _segment_trace(case, log_n, kind, guard=None):
    t = G.rand_matrix(case.width, 1 << log_n, log_n) if kind == "random" else G.edge_matrix(case.width, 1 << log_n, log_n)
    if guard is not None:
        t[guard] = 0
    return t


@pytest.mark.parametrize("kind", ["random", "edge"])
@pytest.mark.parametrize("name", list(BUSES))
def test_segment_proof_with_generated_interactions(ctx, orc, name, kind):
    """interactions only: the LogUp constraints hold for any trace, so the verifier's identity at zeta holds too"""
    case = BUSES[name]
    log_n = 5
    trace = _segment_trace(case, log_n, kind)
    bus = case.bus_program()
    ref = orc.prove(trace, [], [], bus)[:3]
    proof = _check_segment(ctx, orc, (trace, [], [], bus), ref=ref)          # equal to the oracle's proof, openings and queries
    assert proof["perm_width"] == 4 * len(G.chunk_starts(case.bus))
    e_perm, e_cum, _ = G.perm_trace(case.bus, trace, proof["logup_alpha"], proof["logup_beta"])
    assert proof["cumulative_sum"] == e_cum
    assert orc.verify_segment([], [], log_n, case.width, proof, ref[1], ref[2], check_constraints=True, bus=bus) == 0


@pytest.mark.parametrize("kind", ["random", "edge"])
@pytest.mark.parametrize("air_name,bus_name", [("literals", "bus_35"), ("modules", "bus_17")])
def test_segment_proof_with_generated_constraints_and_interactions(ctx, orc, air_name, bus_name, kind):
    """the generated constraints times a guard column next to generated interactions; the trace's guard column is 0, so every
    constraint holds and the proof passes the verifier's identity at zeta"""
    air, buses = AIRS[air_name], BUSES[bus_name]
    guard = air.width - 1
    cons, raw = G.guarded(air, guard)
    case = G.Case(air_name + "+" + bus_name, air.width, cons, raw, buses.bus)
    bc, spans = case.program()
    bus = case.bus_program()
    log_n = 5
    trace = _segment_trace(case, log_n, kind, guard)
    ref = orc.prove(trace, bc, spans, bus)[:3]
    proof = _check_segment(ctx, orc, (trace, bc, spans, bus), ref=ref)
    assert orc.verify_segment(bc, spans, log_n, case.width, proof, ref[1], ref[2], check_constraints=True, bus=bus) == 0


def test_chips_proof_with_a_generated_chip_among_synthetic_ones(ctx, orc):
    gen = BUSES["bus_16"]
    air = AIRS["literals"]
    case = G.Case("literals+bus_16", air.width, air.constraints, air.raw, gen.bus)
    bc, spans = case.program()
    chips = _chips([(6, 12, 0, 7), (4, 9, 2, 3)], seed=21)
    chips.insert(1, (G.edge_matrix(case.width, 1 << 5, 9), bc, spans, case.bus_program()))
    _check_chips(ctx, orc, chips)


@pytest.mark.parametrize("name", [r[0] for r in G.refusal_cases()])
def test_refusals_at_air_creation(ctx, name):
    from powdr_b200 import machine as M
    from powdr_b200.capi import PbError
    _, cons, bus, code = next(r for r in G.refusal_cases() if r[0] == name)
    mach = M.SymbolicMachine(cons)
    bc, spans = M.compile_constraints(mach)
    n0 = ctx.launch_count()
    with pytest.raises(PbError) as err:
        ctx.air(bc, spans, mach.width if cons else 20, bus)
    assert err.value.code == code and ctx.launch_count() == n0


def test_generated_periphery_interactions_match_the_oracle(ctx, orc):
    """variable range checker, tuple range checker and bitwise lookup interactions whose arguments fold and multiply constants (and stay
    inside the tables), with literal, constant-folded, column and quadratic multiplicities, among interactions on other buses"""
    H, num_calls = 1024, 1000
    rng = np.random.default_rng(31)
    tr = np.zeros((6, H), dtype=np.uint32)
    tr[0] = rng.integers(0, 1 << 16, H)          # value
    tr[1] = rng.integers(0, 256, H)              # byte
    tr[2] = rng.integers(0, 256, H)              # byte
    tr[3] = rng.integers(0, 4, H)                # multiplicity
    tr[4] = rng.integers(0, 256, H)
    tr[5] = rng.integers(0, 2048, H)
    tr[:, ::7] = 0
    v, b, c, m, t, s = (G.x(i) for i in range(6))
    one = [P - 1, "*", P - 1]                    # folds to 1
    half = [2, "*", (P + 1) // 2]                # folds to 1
    zero = [[3, "-", 3], "*", 5]                 # folds to 0
    from powdr_b200 import machine as M
    mach = M.SymbolicMachine([], [
        {"id": 3, "mult": m, "args": [[v, "*", one], [[2, "*", 8], "+", 1]]},                   # 16-bit value, max_bits 17
        {"id": 3, "mult": [3, "-", 1], "args": [[[v, "+", 5], "-", [2, "+", 3]], 16]},
        {"id": 3, "mult": [m, "*", m], "args": [[b, "*", half], [8, "*", one]]},
        {"id": 3, "mult": 0, "args": [v, 17]},
        {"id": 6, "mult": m, "args": [[b, "+", zero], [one, "*", c], 0, zero]},                # range: selector folds to 0
        {"id": 6, "mult": 1, "args": [b, [c, "-", zero], 0, one]},                              # xor: selector folds to 1
        {"id": 6, "mult": ["-", [P - 1, "*", m]], "args": [[half, "*", c], b, 0, [P - 1, "*", [P - 1, "*", 1]]]},
        {"id": 7, "mult": m, "args": [[t, "*", one], [[s, "+", 7], "-", 7]]},
        {"id": 7, "mult": [[1 << 27, "*", 15], "*", [P - 1, "*", 2]], "args": [t, [s, "*", half]]},   # (P-1) * (P-2) = 2
        {"id": 1, "mult": 1, "args": [v, [b, "*", 9], 3]},                                      # not a periphery bus
        {"id": 0, "mult": P - 1, "args": []},
    ])
    var_h, t2_h, bw_h = _bus_case(ctx, orc, mach, tr, num_calls)
    assert var_h.sum() > 0 and t2_h.sum() > 0 and bw_h[:65536].sum() > 0 and bw_h[65536:].sum() > 0
