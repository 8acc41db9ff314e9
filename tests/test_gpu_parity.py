"""GPU parity: every CUDA stage, called through the C ABI, against the CPU oracle on the same seeded inputs (bit-exact)."""
import ctypes as C
import os

import numpy as np
import pytest

from util import P, rand_field

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _machine():
    from powdr_b200 import machine
    return machine


# ---------------------------------------------------------------- field / representation
def test_monty_roundtrip(ctx):
    rng = np.random.default_rng(7)
    a = rand_field(rng, 10007)
    a[:4] = [0, 1, P - 1, 2]
    buf = ctx.alloc(a.nbytes).upload(a)
    ctx.lib.pb_to_monty(ctx.h, C.c_void_p(buf.ptr), C.c_size_t(a.size))
    m = buf.download(a.shape)
    assert (m == ((a.astype(np.uint64) << np.uint64(32)) % np.uint64(P)).astype(np.uint32)).all()
    ctx.lib.pb_from_monty(ctx.h, C.c_void_p(buf.ptr), C.c_size_t(a.size))
    assert (buf.download(a.shape) == a).all()


# ---------------------------------------------------------------- stage 1
@pytest.mark.parametrize("log_n,width", [(1, 3), (2, 1), (4, 5), (7, 9), (10, 33), (11, 6), (12, 4), (13, 7), (14, 3), (15, 3), (16, 5), (17, 2)])
def test_lde_matches_oracle(ctx, orc, log_n, width):
    rng = np.random.default_rng(100 + log_n)
    n = 1 << log_n
    trace = rand_field(rng, (width, n))
    d_in = ctx.to_device(trace)
    d_out = ctx.alloc(4 * width * 2 * n)
    ctx.lde_batch(d_in.ptr, log_n, width, d_out.ptr, 1, 31)
    got = ctx.to_host(d_out, (width, 2 * n))
    exp = orc.lde_batch(trace, 1, 31)
    assert (got == exp).all()


@pytest.mark.parametrize("log_blowup,shift", [(2, 31), (1, 1), (1, 1234567), (3, 31)])
def test_lde_blowups_and_shifts(ctx, orc, log_blowup, shift):
    rng = np.random.default_rng(5)
    log_n, width = 9, 6
    trace = rand_field(rng, (width, 1 << log_n))
    d_in = ctx.to_device(trace)
    d_out = ctx.alloc(4 * width * (1 << (log_n + log_blowup)))
    ctx.lde_batch(d_in.ptr, log_n, width, d_out.ptr, log_blowup, shift)
    got = ctx.to_host(d_out, (width, 1 << (log_n + log_blowup)))
    assert (got == orc.lde_batch(trace, log_blowup, shift)).all()


# ---------------------------------------------------------------- stage 3a
def test_poseidon2_permutation(ctx, orc):
    rng = np.random.default_rng(11)
    st = rand_field(rng, (300, 16))
    st[0] = 0
    st[1] = P - 1
    d = ctx.to_device(st)
    ctx.poseidon2_permute(d.ptr, st.shape[0], 1)
    got = ctx.to_host(d, st.shape)
    exp = np.stack([orc.poseidon2_permute(s) for s in st])
    assert (got == exp).all()


def test_poseidon2_plonky3_kat(ctx):
    """CUDA permutation against Plonky3's unit-test vector of default_babybear_poseidon2_16 (input 0..15); provenance of the
    expected words in tests/test_oracle.py::test_poseidon2_plonky3_default_known_answer"""
    exp = [1906786279, 1737026427, 1959749225, 700325316, 1638050605, 1021608788, 1726691001, 1761127344, 1552405120, 417318995,
           36799261, 1215172152, 614923223, 1300746575, 957311597, 304856115]
    st = np.arange(16, dtype=np.uint32).reshape(1, 16)
    d = ctx.to_device(st)
    ctx.poseidon2_permute(d.ptr, 1, 1)
    assert ctx.to_host(d, st.shape)[0].tolist() == exp


def test_poseidon2_custom_constants_generic_diagonal():
    """pb_ctx_set_poseidon2 with arbitrary constants takes the generic (all-Shoup) internal layer; own context so the
    session-wide constants stay untouched"""
    import powdr_b200
    from oracle import orc
    ctx2 = powdr_b200.Context(0)
    try:
        rng = np.random.default_rng(12)
        rc_ext, rc_int, diag = rand_field(rng, (8, 16)), rand_field(rng, 13), rand_field(rng, 16)
        diag[0] = 0
        diag[1] = P - 1
        rc = ctx2.lib.pb_ctx_set_poseidon2(ctx2.h, rc_ext.ctypes.data_as(C.c_void_p), rc_int.ctypes.data_as(C.c_void_p),
                                           diag.ctypes.data_as(C.c_void_p))
        assert rc == 0
        st = rand_field(rng, (64, 16))
        d = ctx2.to_device(st)
        ctx2.poseidon2_permute(d.ptr, st.shape[0], 1)
        got = ctx2.to_host(d, st.shape)
        exp = np.stack([orc.poseidon2_permute_with(s, rc_ext, rc_int, diag) for s in st])
        assert (got == exp).all()
        # restore the default instantiation (device constants are per process, not per context)
        import json
        doc = json.load(open(os.path.join(os.path.dirname(GOLDEN), "..", "constants", "poseidon2_babybear_w16.json")))
        e = np.array(doc["external_initial"] + doc["external_terminal"], dtype=np.uint32)
        i = np.array(doc["internal"], dtype=np.uint32)
        dg = np.array(doc["internal_diag_m1"], dtype=np.uint32)
        assert ctx2.lib.pb_ctx_set_poseidon2(ctx2.h, e.ctypes.data_as(C.c_void_p), i.ctypes.data_as(C.c_void_p), dg.ctypes.data_as(C.c_void_p)) == 0
        st2 = rand_field(rng, (8, 16))
        d2 = ctx2.to_device(st2)
        ctx2.poseidon2_permute(d2.ptr, 8, 1)
        assert (ctx2.to_host(d2, st2.shape) == np.stack([orc.poseidon2_permute(s) for s in st2])).all()
    finally:
        ctx2.close()


@pytest.mark.parametrize("widths,log_h", [([1], 0), ([8], 1), ([3], 3), ([17], 5), ([8, 8], 6), ([4, 4], 11), ([5, 2, 9], 4), ([33], 12)])
def test_merkle_matches_oracle(ctx, orc, widths, log_h):
    rng = np.random.default_rng(13 + log_h)
    h = 1 << log_h
    mats = [rand_field(rng, (w, h)) for w in widths]
    d_mats = [ctx.to_device(m) for m in mats]
    d_layers = ctx.alloc(32 * (2 * h))
    root = ctx.merkle_commit([d.ptr for d in d_mats], widths, log_h, d_layers.ptr)
    got = ctx.to_host(d_layers, (2 * h - 1, 8))
    exp = np.concatenate(orc.merkle_commit(mats))
    assert (got == exp).all()
    assert root == list(exp[-1])


def test_merkle_rows8(ctx, orc):
    rng = np.random.default_rng(17)
    log_h = 9
    rows = rand_field(rng, (1 << log_h, 8))
    d = ctx.to_device(rows)
    d_layers = ctx.alloc(32 * (2 << log_h))
    root = ctx.merkle_commit_rows8(d.ptr, log_h, d_layers.ptr)
    exp = orc.merkle_commit([np.ascontiguousarray(rows.T)])
    assert root == list(exp[-1][0])


def test_merkle_path_verifies_at_scale(ctx, orc):
    """size-independent property: at 2^17 leaves x 40 columns, recompute a few authentication paths on the CPU."""
    rng = np.random.default_rng(19)
    log_h, w = 17, 40
    h = 1 << log_h
    mat = rand_field(rng, (w, h))
    d = ctx.to_device(mat)
    d_layers = ctx.alloc(32 * 2 * h)
    root = ctx.merkle_commit([d.ptr], [w], log_h, d_layers.ptr)
    layers = ctx.to_host(d_layers, (2 * h - 1, 8))
    for r in (0, 1, 77777, h - 1):
        node = orc.hash_row(mat[:, r])
        off, idx, size = 0, r, h
        assert (layers[off + idx] == node).all()
        while size > 1:
            sib = layers[off + (idx ^ 1)]
            node = orc.compress(node, sib) if idx % 2 == 0 else orc.compress(sib, node)
            off += size
            size >>= 1
            idx >>= 1
        assert list(node) == root


# ---------------------------------------------------------------- stage 2
def _compile(ctx, mach):
    m = _machine()
    bc, spans = m.compile_constraints(mach)
    return ctx.air(bc, spans, mach.width), bc, spans


def test_constraint_fold_fixture_single_div(ctx, orc):
    path = os.path.join(GOLDEN, "single_div_nondet.machine.json")
    mach = _machine().SymbolicMachine.from_json_file(path)
    air, bc, spans = _compile(ctx, mach)
    rng = np.random.default_rng(23)
    h = 1000
    mat = rand_field(rng, (mach.width, h))
    mat[:, 0] = 0
    alpha = rand_field(rng, 4)
    d = ctx.to_device(mat)
    d_out = ctx.alloc(16 * h)
    ctx.constraint_fold(air, d.ptr, h, alpha, d_out.ptr)
    got = ctx.to_host(d_out, (4, h))
    exp = orc.constraint_fold(bc, spans, mat, alpha)
    assert (got == exp).all()


@pytest.mark.parametrize("log_n,width,ncons", [(3, 5, 2), (8, 37, 11), (12, 150, 20)])
def test_quotient_matches_oracle(ctx, orc, log_n, width, ncons):
    mach = _machine().synthetic_machine(width, ncons, seed=log_n)
    air, bc, spans = _compile(ctx, mach)
    rng = np.random.default_rng(29)
    n = 1 << log_n
    lde = rand_field(rng, (mach.width, 2 * n))
    alpha = rand_field(rng, 4)
    d = ctx.to_device(lde)
    d_q = ctx.alloc(4 * 8 * n)
    ctx.quotient(air, d.ptr, log_n, alpha, d_q.ptr)
    got = ctx.to_host(d_q, (2, 4, n))
    exp = orc.quotient(bc, spans, lde, log_n, alpha)
    assert (got == exp).all()


def test_bad_bytecode_is_rejected(ctx):
    from powdr_b200.capi import PbError
    with pytest.raises(PbError) as e:
        ctx.air([0, 5], [(0, 2)], 3)             # column 5 >= width 3
    assert e.value.code == -4
    deep = []
    for _ in range(17):
        deep += [1, 1]
    deep += [2] * 16
    with pytest.raises(PbError) as e:
        ctx.air(deep, [(0, len(deep))], 1)       # needs 17 stack slots
    assert e.value.code == -3


# ---------------------------------------------------------------- stage 3b
@pytest.mark.parametrize("log_len", [1, 2, 5, 10, 15])
def test_fri_fold_matches_oracle(ctx, orc, log_len):
    rng = np.random.default_rng(31 + log_len)
    f = rand_field(rng, (1 << log_len, 4))
    beta = rand_field(rng, 4)
    shift = 31 if log_len % 2 else 961
    d = ctx.to_device(f)
    d_out = ctx.alloc(16 * (1 << (log_len - 1)) + 16)
    ctx.fri_fold(d.ptr, log_len, shift, beta, d_out.ptr)
    got = ctx.to_host(d_out, (1 << (log_len - 1), 4))
    assert (got == orc.fri_fold(f, shift, beta)).all()


# ---------------------------------------------------------------- whole segment
@pytest.mark.parametrize("log_n,width,ncons", [(4, 6, 3), (10, 40, 9), (13, 22, 7)])
def test_prove_segment_matches_oracle(ctx, orc, log_n, width, ncons):
    mach = _machine().synthetic_machine(width, ncons, seed=3)
    air, bc, spans = _compile(ctx, mach)
    rng = np.random.default_rng(37)
    trace = rand_field(rng, (mach.width, 1 << log_n))
    exp, _ = orc.prove_segment(trace, bc, spans)
    # device-resident trace
    d = ctx.to_device(trace)
    got = ctx.prove_segment(air, d.ptr, log_n, mach.width, on_device=True)
    assert got == exp
    # host trace (Montgomery form, as a DeviceMatrix transport would hold it)
    from powdr_b200.capi import R_MOD_P
    host = ((trace.astype(np.uint64) * np.uint64(R_MOD_P)) % np.uint64(P)).astype(np.uint32)
    got2 = ctx.prove_segment(air, host.ctypes.data, log_n, mach.width, on_device=False)
    assert got2 == exp
    assert ctx.launch_count() > 0


def test_prove_segment_golden(ctx):
    """committed fixture generated by tests/golden/make_golden.py from the oracle"""
    import json
    with open(os.path.join(GOLDEN, "segment_2p8_w12.json")) as f:
        g = json.load(f)
    mach = _machine().synthetic_machine(g["width"], g["n_constraints"], seed=g["seed"])
    air, bc, spans = _compile(ctx, mach)
    rng = np.random.default_rng(g["trace_seed"])
    trace = rand_field(rng, (mach.width, 1 << g["log_n"]))
    d = ctx.to_device(trace)
    got = ctx.prove_segment(air, d.ptr, g["log_n"], mach.width, on_device=True)
    assert got == g["proof"]


def test_satisfying_trace_gives_low_degree_quotient(ctx):
    """domain property at scale (2^16 rows): an all-zero (padding) trace satisfies every guarded constraint, so the
    quotient is identically zero and the FRI final polynomial is constant zero."""
    mach = _machine().synthetic_machine(64, 12, seed=5)
    air, bc, spans = _compile(ctx, mach)
    log_n = 16
    d = ctx.alloc(4 * mach.width << log_n).zero()
    got = ctx.prove_segment(air, d.ptr, log_n, mach.width, on_device=True)
    assert all(v == [0, 0, 0, 0] for v in got["final_poly"])
    assert got["n_fri_layers"] == log_n


# ---------------------------------------------------------------- stage 2: generated kernel vs interpreter kernel
def test_air_jit_and_interpreter_agree_with_oracle(ctx, orc, monkeypatch):
    """the NVRTC-generated straight-line evaluator and the bytecode interpreter kernel are both CUDA paths of stage 2;
    both must match the oracle on the reference fixture (incl. an INV_OR_ZERO expression)"""
    m = _machine()
    mach = m.SymbolicMachine.from_json_file(os.path.join(GOLDEN, "wasm_register_reuse.machine.json"))
    bc, spans = m.compile_constraints(mach)
    bc = bc + [0, 0, 6, 0, 1, 4]                 # extra constraint: inv_or_zero(col0) * col1
    spans = spans + [(len(bc) - 6, 6)]
    rng = np.random.default_rng(53)
    log_n = 9
    lde = rand_field(rng, (mach.width, 2 << log_n))
    lde[0, :5] = 0
    alpha = rand_field(rng, 4)
    exp = orc.quotient(bc, spans, lde, log_n, alpha)
    d = ctx.to_device(lde)
    d_q = ctx.alloc(4 * 8 << log_n)
    air_jit = ctx.air(bc, spans, mach.width)
    assert air_jit.is_jit
    ctx.quotient(air_jit, d.ptr, log_n, alpha, d_q.ptr)
    assert (ctx.to_host(d_q, (2, 4, 1 << log_n)) == exp).all()
    monkeypatch.setenv("PB_AIR_NO_JIT", "1")
    air_int = ctx.air(bc, spans, mach.width)
    assert not air_int.is_jit
    d_q.zero()
    ctx.quotient(air_int, d.ptr, log_n, alpha, d_q.ptr)
    assert (ctx.to_host(d_q, (2, 4, 1 << log_n)) == exp).all()


def test_host_pipeline_with_many_chunks_matches_device_path(ctx, orc, monkeypatch):
    """the host-input path streams column chunks (PCIe copy || LDE || sponge absorption with states parked in HBM);
    force 8-column chunks so a 43-column trace takes 6 chunks incl. a ragged last one"""
    mach = _machine().synthetic_machine(43, 9, seed=11)
    air, bc, spans = _compile(ctx, mach)
    rng = np.random.default_rng(59)
    log_n = 11
    trace = rand_field(rng, (mach.width, 1 << log_n))
    exp, _ = orc.prove_segment(trace, bc, spans)
    from powdr_b200.capi import R_MOD_P
    host = ((trace.astype(np.uint64) * np.uint64(R_MOD_P)) % np.uint64(P)).astype(np.uint32)
    monkeypatch.setenv("PB_PIPE_CHUNK_COLS", "8")
    got = ctx.prove_segment(air, host.ctypes.data, log_n, mach.width, on_device=False)
    assert got == exp
    monkeypatch.setenv("PB_PIPE_CHUNK_COLS", "16")
    assert ctx.prove_segment(air, host.ctypes.data, log_n, mach.width, on_device=False) == exp


def test_host_pipeline_ramped_schedule_with_ragged_tail(ctx, orc, monkeypatch):
    """wide traces use the ramp-up / ramp-down chunk schedule (8, 16, 32, cw..., 32, 16, 8 + width % 8): 150 columns with
    8-column chunks = 3 + 4 + 3 chunks, the last one 14 columns wide"""
    mach = _machine().synthetic_machine(150, 12, seed=13)
    air, bc, spans = _compile(ctx, mach)
    rng = np.random.default_rng(67)
    log_n = 8
    trace = rand_field(rng, (mach.width, 1 << log_n))
    exp, _ = orc.prove_segment(trace, bc, spans)
    from powdr_b200.capi import R_MOD_P
    host = ((trace.astype(np.uint64) * np.uint64(R_MOD_P)) % np.uint64(P)).astype(np.uint32)
    monkeypatch.setenv("PB_PIPE_CHUNK_COLS", "8")
    assert mach.width >= 4 * 8 + 112 and mach.width % 8 != 0
    assert ctx.prove_segment(air, host.ctypes.data, log_n, mach.width, on_device=False) == exp


# ---------------------------------------------------------------- openings + reduced opening (SURVEY §8f-4)
@pytest.mark.parametrize("log_n,width,shift", [(3, 2, 1), (9, 13, 31), (12, 21, 1234567), (16, 9, 1)])
def test_eval_at_point_matches_oracle(ctx, orc, log_n, width, shift):
    rng = np.random.default_rng(61 + log_n)
    mat = rand_field(rng, (width, 1 << log_n))
    zeta = rand_field(rng, 4)
    d = ctx.to_device(mat)
    d_ys = ctx.alloc(16 * width)
    ctx.eval_at_point(d.ptr, log_n, width, shift, zeta, d_ys.ptr)
    got = ctx.to_host(d_ys, (width, 4))
    assert (got == orc.eval_at_point(mat, shift, zeta)).all()


@pytest.mark.parametrize("log_m,widths", [(4, [3]), (10, [7, 4, 4]), (13, [30, 8])])
def test_deep_quotient_matches_oracle(ctx, orc, log_m, widths):
    rng = np.random.default_rng(67 + log_m)
    m = 1 << log_m
    mats = [rand_field(rng, (w, m)) for w in widths]
    ys = rand_field(rng, (sum(widths), 4))
    zeta, gamma = rand_field(rng, 4), rand_field(rng, 4)
    d_mats = [ctx.to_device(x) for x in mats]
    d_ys = ctx.to_device(ys)
    d_out = ctx.alloc(16 * m)
    ctx.deep_quotient([d.ptr for d in d_mats], widths, log_m, 31, zeta, gamma, d_ys.ptr, d_out.ptr)
    got = ctx.to_host(d_out, (m, 4))
    assert (got == orc.deep_quotient(mats, 31, zeta, gamma, ys)).all()


def test_reduced_opening_is_low_degree_at_scale(ctx):
    """FRI's own invariant as a size-independent property (2^17 rows): for ANY trace the reduced opening
    sum_j gamma^j (f_j(x) - f_j(zeta))/(x - zeta) is a polynomial of degree < N, so after log2(N) folds of the rate-1/2
    codeword the two surviving evaluations are equal (constant final polynomial)"""
    mach = _machine().synthetic_machine(24, 6, seed=13)
    air, bc, spans = _compile(ctx, mach)
    log_n = 17
    rng = np.random.default_rng(71)
    trace = rand_field(rng, (mach.width, 1 << log_n))
    d = ctx.to_device(trace)
    got = ctx.prove_segment(air, d.ptr, log_n, mach.width, on_device=True)
    assert got["final_len"] == 2 and got["final_poly"][0] == got["final_poly"][1]
    assert got["final_poly"][0] != [0, 0, 0, 0]


# ---------------------------------------------------------------- query phase + independent verification
@pytest.mark.parametrize("log_n,width,ncons", [(5, 7, 3), (11, 30, 8)])
def test_gpu_proof_and_queries_match_oracle_and_verify(ctx, orc, log_n, width, ncons):
    mach = _machine().synthetic_machine(width, ncons, seed=17)
    air, bc, spans = _compile(ctx, mach)
    trace = rand_field(np.random.default_rng(83), (mach.width, 1 << log_n))
    d = ctx.to_device(trace)
    ctx.set_fri_params(12, 9)
    try:
        proof = ctx.prove_segment(air, d.ptr, log_n, mach.width, on_device=True)
        queries, ys = ctx.query_segment(log_n, mach.width)
    finally:
        ctx.set_fri_params(8, 4)
    exp_proof, exp_ys, exp_q = orc.prove_segment_q(trace, bc, spans, 12, pow_bits=9)
    assert proof == exp_proof and (ys == exp_ys).all() and (queries == exp_q).all()
    assert orc.verify_segment(bc, spans, log_n, mach.width, proof, ys, queries) == 0


def test_gpu_proof_of_a_satisfying_trace_verifies_with_the_constraint_identity(ctx, orc):
    """the reference's own notion of correctness: the GPU engine's proof verifies under the CPU verifier"""
    from powdr_b200 import machine as M
    mach = M.SymbolicMachine([["b@0", "*", ["b@0", "-", 1]], [["b@0", "*", "c@1"], "-", "d@2"]])
    air, bc, spans = _compile(ctx, mach)
    log_n = 14
    rng = np.random.default_rng(89)
    b = rng.integers(0, 2, 1 << log_n).astype(np.uint32)
    c = rand_field(rng, 1 << log_n)
    dd = (b.astype(np.uint64) * c % P).astype(np.uint32)
    trace = np.stack([b, c, dd])
    dev = ctx.to_device(trace)
    proof = ctx.prove_segment(air, dev.ptr, log_n, 3, on_device=True)
    queries, ys = ctx.query_segment(log_n, 3)
    assert orc.verify_segment(bc, spans, log_n, 3, proof, ys, queries, check_constraints=True) == 0
    trace[1, 5] = (int(trace[1, 5]) + 1) % P if b[5] else trace[1, 5]
    trace[2, 9] = (int(trace[2, 9]) + 1) % P
    dev = ctx.to_device(trace)
    proof = ctx.prove_segment(air, dev.ptr, log_n, 3, on_device=True)
    queries, ys = ctx.query_segment(log_n, 3)
    assert orc.verify_segment(bc, spans, log_n, 3, proof, ys, queries, check_constraints=False) == 0
    assert orc.verify_segment(bc, spans, log_n, 3, proof, ys, queries, check_constraints=True) == 16


# ---------------------------------------------------------------- LogUp / bus-interaction argument (SURVEY §8 f1)
@pytest.mark.parametrize("log_n,width,n_ints,quad,ncons", [(3, 12, 5, 0, 0), (7, 20, 9, 3, 4), (10, 33, 40, 7, 6), (12, 10, 1, 0, 2)])
def test_logup_segment_matches_oracle_and_verifies(ctx, orc, log_n, width, n_ints, quad, ncons):
    """bus interactions attached to the AIR: permutation trace, running sum, LogUp constraints in the quotient, two opening
    points -- proof, opened values and query openings bit-identical to the oracle's; the independent verifier accepts"""
    M = _machine()
    base = M.synthetic_machine(width, ncons, seed=3) if ncons else None
    mach = M.SymbolicMachine(base.constraints if base else [], M.synthetic_bus(width, n_ints, 10 + log_n, quad))
    bc, spans = M.compile_constraints(mach)
    bus = M.compile_bus(mach, 1)
    air = ctx.air(bc, spans, mach.width, bus)
    assert air.perm_width > 0
    rng = np.random.default_rng(log_n)
    trace = rand_field(rng, (mach.width, 1 << log_n))
    d = ctx.to_device(trace)
    proof = ctx.prove_segment(air, d.ptr, log_n, mach.width, on_device=True)
    queries, ys = ctx.query_segment(log_n, mach.width, air.perm_width)
    exp_proof, exp_ys, exp_q, _ = orc.prove(trace, bc, spans, bus, n_queries=8, pow_bits=4)
    assert proof["perm_width"] == air.perm_width == exp_proof["perm_width"]
    assert proof["cumulative_sum"] == exp_proof["cumulative_sum"] and proof["perm_root"] == exp_proof["perm_root"]
    assert proof["quotient_root"] == exp_proof["quotient_root"]
    assert proof == exp_proof and (ys == exp_ys).all() and (queries == exp_q).all()
    assert orc.verify_segment(bc, spans, log_n, mach.width, proof, ys, queries, check_constraints=(ncons == 0), bus=bus) == 0
    # host-resident trace takes the pipelined commit, then the same LogUp phase
    from powdr_b200.capi import R_MOD_P
    host = ((trace.astype(np.uint64) * np.uint64(R_MOD_P)) % np.uint64(P)).astype(np.uint32)
    assert ctx.prove_segment(air, host.ctypes.data, log_n, mach.width, on_device=False) == exp_proof


def test_logup_at_scale_verifies(ctx, orc):
    """2^15 rows x 300 interactions (150+ chunks, several JIT groups): too slow for the scalar oracle prover, so the check is
    the independent verifier (all challenges, proof of work, 8 queries with three Merkle paths each, folds) plus the LogUp
    identity at zeta, which holds for ANY trace when the AIR has interactions only"""
    M = _machine()
    mach = M.SymbolicMachine([], M.synthetic_bus(96, 300, 77, quadratic_every=11))
    bus = M.compile_bus(mach, 1)
    air = ctx.air([], [], mach.width, bus)
    log_n = 15
    trace = rand_field(np.random.default_rng(15), (mach.width, 1 << log_n))
    d = ctx.to_device(trace)
    proof = ctx.prove_segment(air, d.ptr, log_n, mach.width, on_device=True)
    queries, ys = ctx.query_segment(log_n, mach.width, air.perm_width)
    assert proof["final_poly"][0] == proof["final_poly"][1]
    assert orc.verify_segment([], [], log_n, mach.width, proof, ys, queries, check_constraints=True, bus=bus) == 0


def test_proof_of_work_default_parameters(orc):
    """default context parameters (100 queries, 16 PoW bits): the GPU grinding kernel finds the same (smallest) witness as the oracle"""
    import powdr_b200
    M = _machine()
    c2 = powdr_b200.Context(0)
    try:
        mach = M.synthetic_machine(9, 3, seed=2)
        bc, spans = M.compile_constraints(mach)
        air = c2.air(bc, spans, mach.width)
        trace = rand_field(np.random.default_rng(16), (mach.width, 1 << 6))
        d = c2.to_device(trace)
        proof = c2.prove_segment(air, d.ptr, 6, mach.width, on_device=True)
        queries, ys = c2.query_segment(6, mach.width)
        exp, exp_ys, exp_q, _ = orc.prove(trace, bc, spans, None, n_queries=100, pow_bits=16)
        assert proof["pow_bits"] == 16 and proof["n_queries"] == 100 and proof["pow_witness"] == exp["pow_witness"]
        assert proof == exp and (queries == exp_q).all()
        assert orc.verify_segment(bc, spans, 6, mach.width, proof, ys, queries) == 0
    finally:
        c2.close()


def test_large_preopt_fixture_jit_chunks_and_interpreter_agree_with_oracle(ctx, orc, monkeypatch):
    """apc_reth_op_bug (5869 columns, 9168 constraints): the JIT splits it into ~70 modules whose kernels pass the running fold
    through a scratch buffer; the interpreter is the other CUDA path.  Both must equal the oracle on random rows."""
    path = os.path.join(GOLDEN, "apc_reth_op_bug.machine.json.gz")
    mach = _machine().SymbolicMachine.from_json_file(path)
    bc, spans = _machine().compile_constraints(mach)
    rng = np.random.default_rng(31)
    h = 200
    mat = rand_field(rng, (mach.width, h))
    alpha = rand_field(rng, 4)
    exp = orc.constraint_fold(bc, spans, mat, alpha)
    d = ctx.to_device(mat)
    d_out = ctx.alloc(16 * h)
    air = ctx.air(bc, spans, mach.width)
    assert air.is_jit
    ctx.constraint_fold(air, d.ptr, h, alpha, d_out.ptr)
    assert (ctx.to_host(d_out, (4, h)) == exp).all()
    monkeypatch.setenv("PB_AIR_NO_JIT", "1")
    interp = ctx.air(bc, spans, mach.width)
    assert not interp.is_jit
    d_out.zero()
    ctx.constraint_fold(interp, d.ptr, h, alpha, d_out.ptr)
    assert (ctx.to_host(d_out, (4, h)) == exp).all()


def test_plain_c_client_produces_the_same_commitments(ctx, orc, tmp_path):
    """examples/abi_demo.c (gcc, no Python in the loop) proves a satisfying 3-column trace from host memory; the Python binding
    and the oracle must produce the same roots, and the FRI final polynomial is a constant"""
    import subprocess
    from test_host import _build_abi_demo
    log_n = 10
    r = subprocess.run([_build_abi_demo(tmp_path), str(log_n)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    out = {ln.split()[0]: ln.split()[1:] for ln in r.stdout.strip().splitlines()}
    n = 1 << log_n
    s, mask = 88172645463325252, (1 << 64) - 1
    trace = np.zeros((3, n), dtype=np.uint32)
    for row in range(n):
        s ^= (s << 13) & mask
        s ^= s >> 7
        s ^= (s << 17) & mask
        a, b = s % 3, (s >> 8) % P
        trace[:, row] = [a, b, a * b % P]
    A, B, Cc = "a@0", "b@1", "c@2"
    from powdr_b200 import machine as M
    mach = M.SymbolicMachine([[[A, "*", B], "-", Cc], [[A, "*", [A, "-", 1]], "*", [A, "-", 2]]], [], [])
    assert mach.width == 3
    bc, spans = M.compile_constraints(mach)
    exp, _ = orc.prove_segment(trace, bc, spans, n_queries=0, pow_bits=0)
    assert [int(x) for x in out["trace_root"]] == exp["trace_root"]
    assert [int(x) for x in out["quotient_root"]] == exp["quotient_root"]
    fin = [int(x) for x in out["fri_layers"][4:]]
    assert int(out["fri_layers"][0]) == exp["n_fri_layers"] and fin == [v for row in exp["final_poly"][:exp["final_len"]] for v in row]
    assert fin[:4] == fin[4:8]                    # constant final polynomial: the quotient of a satisfying trace is low degree
