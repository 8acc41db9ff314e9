"""The generated AIRs of tests/exprgen.py on the CPU: the oracle's constraint fold, quotient and LogUp permutation trace against the
plain evaluator, the code generators' NVRTC output for sm_90a (compile only, no device), and the refusal codes of the entry points."""
import ctypes as C
import glob
import re

import numpy as np
import pytest

import exprgen as G
from util import P, rand_field

AIRS = {c.name: c for c in G.all_air_cases()}
BUSES = {c.name: c for c in G.bus_cases()}
ALPHA = [123456789, 987654321, 5, P - 1]


def _lib():
    import powdr_b200
    return powdr_b200.load_library()


def _spans(spans):
    from powdr_b200.capi import Span
    sp = (Span * max(1, len(spans)))()
    for i, (o, l) in enumerate(spans):
        sp[i].off, sp[i].len = o, l
    return sp


def air_compile_only(bc, spans, width):
    b = np.ascontiguousarray(bc, dtype=np.uint32)
    sz = C.c_size_t()
    rc = _lib().pb_air_jit_compile_only(b.ctypes.data_as(C.c_void_p), C.c_size_t(b.size), _spans(spans), C.c_size_t(len(spans)),
                                         C.c_uint32(width), C.byref(sz))
    return rc, sz.value


def _bus_args(bus, width):
    from powdr_b200 import capi
    ints, isp, ibc = bus
    ibc = np.ascontiguousarray(ibc, dtype=np.uint32)
    di = (capi.DevInteraction * max(1, len(ints)))()
    for i, (b, n, o) in enumerate(ints):
        di[i].bus_id, di[i].num_args, di[i].args_index_off = b, n, o
    return (ibc, ibc.ctypes.data_as(C.c_void_p), C.c_size_t(ibc.size), _spans(isp), C.c_size_t(len(isp)), di, C.c_size_t(len(ints)),
            C.c_uint32(width))


def logup_compile_only(bus, width):
    keep, *args = _bus_args(bus, width)
    cb, wp = C.c_size_t(), C.c_size_t()
    rc = _lib().pb_air_logup_compile_only(*args, C.byref(cb), C.byref(wp))
    return rc, wp.value


def _traces(width, n, seed):
    return {"random": G.rand_matrix(width, n, seed), "edge": G.edge_matrix(width, n, seed)}


# ---------------------------------------------------------------- the oracle against the evaluator
@pytest.mark.parametrize("name", list(AIRS))
def test_oracle_fold_and_quotient_agree_with_the_evaluator(orc, name):
    case = AIRS[name]
    bc, spans = case.program()
    for kind, mat in _traces(case.width, 64, 3).items():
        assert (orc.constraint_fold(bc, spans, mat, ALPHA) == case.fold(mat, ALPHA)).all(), kind
    log_n = 5
    for kind, lde in _traces(case.width, 2 << log_n, 4).items():
        exp = G.quotient(case.fold(lde, ALPHA), log_n)
        assert (orc.quotient(bc, spans, lde, log_n, ALPHA) == exp).all(), kind


def test_evaluator_folds_the_inverse_cases_by_hand():
    """the raw OP_INV_OR_ZERO constraints on a row where their columns are 0 and on one where they are 3"""
    case = AIRS["literals"]
    mat = np.zeros((case.width, 2), dtype=np.uint32)
    mat[:, 1] = 3
    i3, i7 = pow(3, P - 2, P), pow(7, P - 2, P)
    exp = [[0, 0, 3, 0, 0, 0, P - 1, 0, 0, 1], [i3, 0, 3, 3, 1, 0, 2, (P - i3) * i7 % P, 3 * pow(2, P - 2, P) % P, 1]]
    for r in range(2):
        assert [int(G.eval_ops(G.ops_of_words(w), mat)[r]) for w in case.raw] == exp[r]


@pytest.mark.parametrize("name", list(BUSES))
def test_oracle_perm_trace_agrees_with_the_evaluator(orc, name):
    case = BUSES[name]
    rng = np.random.default_rng(7)
    al, be = rand_field(rng, 4).tolist(), rand_field(rng, 4).tolist()
    for kind, trace in _traces(case.width, 8, 5).items():
        perm, cum, cs = orc.logup_perm_trace(trace, case.bus_program(), al, be)
        e_perm, e_cum, e_cs = G.perm_trace(case.bus, trace, al, be)
        assert cs == e_cs
        assert (perm == e_perm).all(), kind
        assert cum.tolist() == e_cum


def test_generated_interactions_reach_every_chunk_shape():
    """what the LogUp generator has to handle occurs in the generated bus cases"""
    sizes, ids, nargs, mults, mdeg = set(), set(), set(), set(), set()
    from powdr_b200 import machine as M
    for case in BUSES.values():
        cs = G.chunk_starts(case.bus)
        sizes.update(b - a for a, b in zip(cs, cs[1:]))
        for b in case.bus:
            ids.add(b["id"])
            nargs.add(len(b["args"]))
            mdeg.add(M.degree(b["mult"]))
            if M.degree(b["mult"]) == 0:
                mults.add(int(G.eval_ops(G.ops_of_tree(b["mult"]), np.zeros((1, 1), dtype=np.uint32))[0]))
    assert {1, 2, 3, 5, 17, 40} <= sizes
    assert {0, P - 1} <= ids and 0 in nargs and max(nargs) > 9
    assert {0, 1, P - 1} <= mults and {0, 1, 2, 3} <= mdeg
    assert {len(G.chunk_starts(c.bus)) - 1 for c in BUSES.values()} == {1, 2, 3, 15, 16, 17, 35}


# ---------------------------------------------------------------- the generators' source, compiled for sm_90a
def _dumps(prefix):
    return [open(f).read() for f in sorted(glob.glob(prefix + ".*.cu"), key=lambda f: int(f.rsplit(".", 2)[1]))]


@pytest.mark.parametrize("name", list(AIRS))
def test_constraint_codegen_compiles_every_generated_air(name, tmp_path, monkeypatch):
    case = AIRS[name]
    bc, spans = case.program()
    monkeypatch.setenv("PB_AIR_JIT_DUMP", str(tmp_path / "air"))
    rc, size = air_compile_only(bc, spans, case.width)
    assert rc == 0 and size > 0
    srcs = _dumps(str(tmp_path / "air"))
    assert len(srcs) == len(G.module_bounds(case)) - 1
    src = "".join(srcs)
    assert "mulc(" in src and " inv(" in src and " neg(" in src
    if name == "modules":
        assert len(srcs) >= 4 and "__ldg(b + " in src                  # columns past the 32 hoisted ones, loaded at use
        assert re.search(r"asm volatile\(\"ld.global.nc.u32 %0, \[%1\];\" : \"=r\"\(c31\)", src)
        g0 = srcs[0].split("__device__ __noinline__ uint4 g")[1:]
        assert len(g0) == 4                                           # 600 | 300 | 301 | 799
    if name == "literals":                                            # constant constraints fold to a literal in the fold call
        assert re.search(r"acc = fold\(acc, 0x[0-9a-f]{8}u, ", src)


@pytest.mark.parametrize("name", list(BUSES))
def test_logup_codegen_compiles_every_generated_bus(name, tmp_path, monkeypatch):
    case = BUSES[name]
    monkeypatch.setenv("PB_LOGUP_JIT_DUMP", str(tmp_path / "lu"))
    rc, wp = logup_compile_only(case.bus_program(), case.width)
    n_chunks = len(G.chunk_starts(case.bus)) - 1
    assert rc == 0 and wp == 4 * (n_chunks + 1)
    srcs = _dumps(str(tmp_path / "lu"))
    assert len(srcs) == -(-n_chunks // G.MODULE_CHUNKS)
    src = "".join(srcs)
    if any(b - a >= 3 for a, b in zip(G.chunk_starts(case.bus), G.chunk_starts(case.bus)[1:])):
        assert re.search(r"N\d+ = e_add\(e_mul\(N\d+, d\d+\), e_scale\(D\d+, ", src)
    keep, *args = _bus_args(case.bus_program(), case.width)
    assert _lib().pb_bus_compile(None, *args, C.c_uint32(3), C.c_uint32(7), C.c_uint32(6), None) == 0


@pytest.mark.parametrize("name", [r[0] for r in G.refusal_cases()])
def test_refusals_return_the_codes_of_the_gpu_entry_points(name):
    from powdr_b200 import machine as M
    _, cons, bus, code = next(r for r in G.refusal_cases() if r[0] == name)
    if cons:
        mach = M.SymbolicMachine(cons)
        bc, spans = M.compile_constraints(mach)
        assert air_compile_only(bc, spans, mach.width)[0] == code
    else:
        assert logup_compile_only(bus, 20)[0] == code


def test_depth_16_is_accepted_in_a_constraint_and_an_interaction():
    from powdr_b200 import machine as M
    mach = M.SymbolicMachine([G.depth_tree(16)], [{"id": 1, "mult": G.x(0), "args": [G.depth_tree(16, 1, "+-")]}])
    bc, spans = M.compile_constraints(mach)
    assert air_compile_only(bc, spans, mach.width)[0] == 0
    assert logup_compile_only(M.compile_bus(mach, 1), mach.width)[0] == 0
