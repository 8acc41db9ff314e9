"""The prover at both ends of its height range (chip_ok: 1 <= log_n <= 24) and at the widths and values where its kernels change path,
against the oracle (oracle/prove.c) bit for bit -- proof, cumulative sums, opened values and query words -- and its verifier:

  * 2- and 4-row chips: the lowest FRI injection (h = 2), a one-layer FRI, Merkle trees of 2 to 4 leaves, openings over fewer rows
    than one CTA, query paths of length 1 and 2, more queries than domain positions;
  * 2^21 to 2^24-row chips: FRI from a 2^25 codeword, eval_at_point with 512 splits, mixed-height trees injecting 22 levels up;
  * openings wider than the gamma-power staging chunk of deep_quotient_kernel (256 columns at one point, 128 at two points);
  * traces of 0, 1, P-1, P-2, alternating 0 / P-1 and single P-1 spikes, with LogUp multiplicities 0 and P-1, on both sides of the
    cooperative Merkle kernels' threshold.

The CPU tests at the top pin the oracle itself at 2 and 4 rows."""
import ctypes as C
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from test_gpu_chips import _chips, _gpu_prove
from util import P, bitrev, rand_field

gpu = pytest.mark.gpu

R_MOD_P = (1 << 32) % P


def _mont(a):
    return ((np.asarray(a, dtype=np.uint32).astype(np.uint64) * np.uint64(R_MOD_P)) % np.uint64(P)).astype(np.uint32)


def _gpu_segment(ctx, chip, on_device=True):
    """pb_prove_segment + pb_query_segment -> (proof, opened values, query words)"""
    trace, bc, spans, bus = chip
    w, n = trace.shape
    log_n = n.bit_length() - 1
    air = ctx.air(bc, spans, w, bus)
    try:
        if on_device:
            d = ctx.to_device(trace)
            proof = ctx.prove_segment(air, d.ptr, log_n, w, on_device=True)
            d.free()
        else:
            host = _mont(trace)
            proof = ctx.prove_segment(air, host.ctypes.data, log_n, w, on_device=False)
        q, ys = ctx.query_segment(log_n, w, air.perm_width)
    finally:
        air.free()
    return proof, ys, q


def _check_segment(ctx, orc, chip, on_device=True, ref=None):
    trace, bc, spans, bus = chip
    proof, ys, q = _gpu_segment(ctx, chip, on_device)
    e_proof, e_ys, e_q = ref if ref is not None else orc.prove(trace, bc, spans, bus)[:3]
    assert proof["trace_root"] == e_proof["trace_root"] and proof["perm_root"] == e_proof["perm_root"]
    assert proof["cumulative_sum"] == e_proof["cumulative_sum"] and proof["quotient_root"] == e_proof["quotient_root"]
    assert (ys == e_ys).all()
    assert proof["fri_roots"] == e_proof["fri_roots"] and proof["final_poly"] == e_proof["final_poly"]
    assert proof == e_proof and (q == e_q).all()
    assert orc.verify_segment(bc, spans, trace.shape[1].bit_length() - 1, trace.shape[0], proof, ys, q, bus=bus) == 0
    return proof


def _check_chips(ctx, orc, chips, ref=None):
    proof, cs, ys, q = _gpu_prove(ctx, chips)
    e_proof, e_cs, e_ys, e_q = ref if ref is not None else orc.prove_chips(chips)
    assert proof["main_root"] == e_proof["main_root"]
    assert (cs == e_cs).all() and proof["perm_root"] == e_proof["perm_root"]
    assert proof["quotient_root"] == e_proof["quotient_root"]
    assert (ys == e_ys).all()
    assert proof["fri_roots"] == e_proof["fri_roots"] and proof["final_poly"] == e_proof["final_poly"]
    assert proof == e_proof and (q == e_q).all()
    assert orc.verify_chips(chips, proof, cs, ys, q, check_constraints=False) == 0
    return proof


# ---------------------------------------------------------------- 1. 2- and 4-row chips
SHORT_SEGMENTS = {                      # variant -> (n_constraints, n_interactions, on_device)
    "constraints_and_interactions": (2, 3, True),
    "interactions_only": (0, 3, True),
    "constraints_only": (2, 0, True),
    "host_trace": (2, 3, False),
}

SHORT_MIXES = {
    "inject_at_h2": [(1, 6, 2, 3), (6, 12, 0, 7)],                      # a 2-row chip next to a 2^6 one: a codeword injected at h = 2
    "rows_2_4_32": [(1, 5, 1, 2), (2, 7, 2, 3), (5, 9, 0, 4)],
    "three_2_row_chips": [(1, 4, 1, 2), (1, 6, 0, 3), (1, 5, 2, 0)],   # one height; the whole proof is a one-layer FRI
    "short_perm_tree": [(1, 5, 0, 4), (7, 12, 3, 0), (5, 8, 2, 0)],     # the 2-row chip alone has interactions: perm tree of 4 leaves
}


def test_oracle_proves_and_verifies_2_and_4_row_segments(orc):
    for log_n in (1, 2):
        for ncons, nints, _ in SHORT_SEGMENTS.values():
            trace, bc, spans, bus = _chips([(log_n, 6, ncons, nints)], seed=log_n)[0]
            proof, ys, q, _ = orc.prove(trace, bc, spans, bus)
            assert proof["n_fri_layers"] == log_n and proof["final_len"] == 2
            assert orc.verify_segment(bc, spans, log_n, trace.shape[0], proof, ys, q, bus=bus) == 0
            if not ncons:                                   # interaction-only: the LogUp identity at zeta holds for any trace
                assert orc.verify_segment(bc, spans, log_n, trace.shape[0], proof, ys, q, check_constraints=True, bus=bus) == 0
            for row in (0, trace.shape[0] - 1, ys.shape[0] - 1):
                y2 = ys.copy()
                y2[row, 1] = (int(y2[row, 1]) + 1) % P
                assert orc.verify_segment(bc, spans, log_n, trace.shape[0], proof, y2, q, bus=bus) != 0
            if orc.fast_available():
                f_proof, f_ys, f_q, _ = orc.prove(trace, bc, spans, bus, fast=True)
                assert f_proof == proof and (f_ys == ys).all() and (f_q == q).all()


@pytest.mark.parametrize("mix", list(SHORT_MIXES))
def test_oracle_proves_and_verifies_short_chip_mixes(orc, mix):
    spec = SHORT_MIXES[mix]
    chips = _chips(spec, seed=11)
    proof, cs, ys, q = orc.prove_chips(chips)
    assert proof["log_max"] == max(s[0] for s in spec) + 1
    assert orc.verify_chips(chips, proof, cs, ys, q, check_constraints=False) == 0
    for i in (0, ys.shape[0] // 2, ys.shape[0] - 1):
        y2 = ys.copy()
        y2[i, 3] = (int(y2[i, 3]) + 1) % P
        assert orc.verify_chips(chips, proof, cs, y2, q, check_constraints=False) != 0
    if orc.fast_available():
        f = orc.prove_chips(chips, fast=True)
        assert f[0] == proof and (f[1] == cs).all() and (f[2] == ys).all() and (f[3] == q).all()


@gpu
@pytest.mark.parametrize("variant", list(SHORT_SEGMENTS))
@pytest.mark.parametrize("log_n", [1, 2])
def test_short_segment_matches_oracle(ctx, orc, log_n, variant):
    ncons, nints, on_device = SHORT_SEGMENTS[variant]
    chip = _chips([(log_n, 6, ncons, nints)], seed=log_n)[0]
    proof = _check_segment(ctx, orc, chip, on_device)
    assert proof["n_fri_layers"] == log_n


@gpu
@pytest.mark.parametrize("mix", list(SHORT_MIXES))
def test_short_chip_mix_matches_oracle(ctx, orc, mix):
    _check_chips(ctx, orc, _chips(SHORT_MIXES[mix], seed=11))


@gpu
def test_2_row_segment_at_default_parameters(orc):
    """100 queries and 16 proof-of-work bits (a fresh context's defaults) on a domain of 4 positions: every position is queried
    many times over"""
    import powdr_b200
    c2 = powdr_b200.Context(0)
    try:
        chip = _chips([(1, 6, 2, 3)], seed=21)[0]
        trace, bc, spans, bus = chip
        proof = _check_segment(c2, orc, chip, ref=orc.prove(trace, bc, spans, bus, n_queries=100, pow_bits=16)[:3])
        assert (proof["n_queries"], proof["pow_bits"]) == (100, 16)
        chips = _chips([(1, 6, 2, 3), (1, 4, 0, 2)], seed=22)
        _check_chips(c2, orc, chips, ref=orc.prove_chips(chips, n_queries=100, pow_bits=16))
    finally:
        c2.close()


@gpu
def test_sharded_chips_refuse_a_2_row_chip_before_any_collective(ctx):
    """a 2-row chip is below the sharded provers' minimum height 2^(g + 3) for every world size"""
    from powdr_b200.capi import Chip, ChipsProof
    from powdr_b200.sharded import Comm, shard_columns

    class NoCollective(Comm):
        called = 0

        def all_gather(self, send, recv, nbytes):
            NoCollective.called += 1
            raise AssertionError("collective called")

        all_to_all = all_gather

    chips = _chips([(6, 12, 2, 3), (1, 4, 1, 2)], seed=5)
    airs = [ctx.air(bc, sp, t.shape[0], bus) for t, bc, sp, bus in chips]
    proof, cs = ChipsProof(), (C.c_uint32 * 8)()
    world = 2
    for rank in range(world):
        blocks = []
        for t, _, _, _ in chips:
            f, n = shard_columns(t.shape[0], world, rank)
            blocks.append(ctx.to_device(t[f:f + n]) if n else None)
        arr = (Chip * 2)(*[Chip(a.h.value, b.ptr if b else None, t.shape[1].bit_length() - 1, t.shape[0])
                           for a, b, (t, _, _, _) in zip(airs, blocks, chips)])
        comm = NoCollective(rank, world)
        assert ctx.lib.pb_prove_chips_sharded(ctx.h, arr, C.c_size_t(2), C.byref(comm.c), C.byref(proof), cs) == -2   # PB_ERR_UNSUPPORTED
    assert NoCollective.called == 0
    for a in airs:
        a.free()


# ---------------------------------------------------------------- 2. 2^21 to 2^24-row chips
TALL_WIDTH, TALL_CONS, TALL_INTS = 6, 2, 3
TALL_SEGMENTS = {"2p21": (21, True), "2p22_host_trace": (22, False), "2p24": (24, True)}
TALL_MIX = [(23, TALL_WIDTH, TALL_CONS, TALL_INTS), (2, 5, 1, 2), (1, 4, 0, 2)]


class TallRefs:
    """The tall chips and, where the AVX-512 oracle arm is available, its proofs of them: all four are started together on first use
    and computed concurrently (ctypes releases the GIL) while the GPU proves; a test waits only for its own."""

    def __init__(self, orc):
        self.segments = {k: _chips([(ln, TALL_WIDTH, TALL_CONS, TALL_INTS)], seed=ln)[0] for k, (ln, _) in TALL_SEGMENTS.items()}
        self.mix = _chips(TALL_MIX, seed=23)
        self.fast = orc.fast_available()
        self._pool = self._futures = None
        if self.fast:
            self._pool = ThreadPoolExecutor(len(TALL_SEGMENTS) + 1)
            self._futures = {k: self._pool.submit(lambda c: orc.prove(c[0], c[1], c[2], c[3], fast=True)[:3], c)
                             for k, c in self.segments.items()}
            self._futures["mix"] = self._pool.submit(lambda: orc.prove_chips(self.mix, fast=True))

    def ref(self, key):
        return self._futures[key].result() if self.fast else None

    def close(self):
        if self._pool is not None:
            self._pool.shutdown(cancel_futures=True)


@pytest.fixture(scope="module")
def tall(orc):
    r = TallRefs(orc)
    yield r
    r.close()


def _sampled_checks(ctx, orc, chip, n_lde_checks):
    """what holds of a proof without the oracle proving it (test_gpu_fullsize.py): the same trace under an interaction-only AIR
    verifies WITH the constraint identity, and under a constraint-only AIR its opened LDE rows are the trace polynomials at the
    queried points and its opened quotient rows are the alpha-fold of the constraints over Z_H"""
    trace, bc, spans, bus = chip
    w, n = trace.shape
    log_n, log_m = n.bit_length() - 1, n.bit_length()
    bus_only = (trace, [], [], bus)
    proof, ys, q = _gpu_segment(ctx, bus_only)
    assert orc.verify_segment([], [], log_n, w, proof, ys, q, check_constraints=True, bus=bus) == 0
    cons_only = (trace, bc, spans, None)
    proof, ys, q = _gpu_segment(ctx, cons_only)
    assert orc.verify_segment(bc, spans, log_n, w, proof, ys, q) == 0
    w_m, g_n = pow(31, (P - 1) >> log_m, P), pow(31, n, P)
    ev_at = orc.fast_eval_at_point if orc.fast_available() else orc.eval_at_point
    for qi in range(q.shape[0]):
        i_nat = bitrev(int(q[qi, 0]), log_m)
        x = 31 * pow(w_m, i_nat, P) % P
        row = q[qi, 1:1 + w]
        qrow = q[qi, 1 + w + 8 * log_m:1 + w + 8 * log_m + 8]
        if qi < n_lde_checks:
            ev = ev_at(trace, 1, [x, 0, 0, 0])
            assert (ev[:, 1:] == 0).all() and (ev[:, 0] == row).all(), qi
        acc = orc.constraint_fold(bc, spans, row.reshape(w, 1), proof["alpha"])[:, 0].tolist()
        par = i_nat & 1
        zh = (g_n * (P - 1 if par else 1) - 1) % P
        assert [int(v) for v in acc] == [zh * int(qrow[4 * par + l]) % P for l in range(4)], qi


@gpu
@pytest.mark.parametrize("key", list(TALL_SEGMENTS))
def test_tall_segment(ctx, orc, tall, key):
    """bit for bit against the AVX-512 oracle arm where it is available; the sampled checks run either way"""
    log_n, on_device = TALL_SEGMENTS[key]
    chip = tall.segments[key]
    if tall.fast:
        proof = _check_segment(ctx, orc, chip, on_device, ref=tall.ref(key))
    else:
        trace, bc, spans, bus = chip
        proof, ys, q = _gpu_segment(ctx, chip, on_device)
        assert orc.verify_segment(bc, spans, log_n, trace.shape[0], proof, ys, q, bus=bus) == 0
    assert proof["n_fri_layers"] == log_n and proof["final_poly"][0] == proof["final_poly"][1]
    _sampled_checks(ctx, orc, chip, n_lde_checks=2 if orc.fast_available() else 1)


@gpu
def test_tall_chip_with_2_and_4_row_chips(ctx, orc, tall):
    """a 2^23-row chip with 4- and 2-row ones: their codewords are injected 21 and 22 folds down the FRI of the 2^24 codeword"""
    if tall.fast:
        proof = _check_chips(ctx, orc, tall.mix, ref=tall.ref("mix"))
    else:
        bus_only = [(t, [], [], bus) for t, _, _, bus in tall.mix]
        proof, cs, ys, q = _gpu_prove(ctx, bus_only)
        assert orc.verify_chips(bus_only, proof, cs, ys, q, check_constraints=True) == 0
        proof, cs, ys, q = _gpu_prove(ctx, tall.mix)
        assert orc.verify_chips(tall.mix, proof, cs, ys, q, check_constraints=False) == 0
    assert proof["log_max"] == 24 and proof["final_poly"][0] == proof["final_poly"][1]


# ---------------------------------------------------------------- 3. openings wider than a staging chunk
def _n_ints_for_perm_width(orc, width, perm_width):
    """the number of synthetic interactions (chip seed 200, as _chips builds them) whose permutation trace is perm_width wide"""
    from powdr_b200 import machine as M
    for k in range(1, 4 * perm_width):
        mach = M.SymbolicMachine([], M.synthetic_bus(width, k, seed=200, quadratic_every=5))
        if orc.Air([], [], M.compile_bus(mach, 1)).perm_width == perm_width:
            return k
    raise AssertionError("no interaction count gives a %d-column permutation trace" % perm_width)


WIDE = {                                    # main widths against DQ_CHUNK = 256, permutation widths against DQ_CHUNK / 2 = 128
    "main_517": [(4, 517, 5, 0)],           # 256 + 256 + 5
    "perm_140_interactions": [(3, 40, 0, 140)],
    "main_and_perm": [(5, 517, 3, 140)],
    "main_tail_3": [(3, 259, 2, 0)],
    "main_tail_13": [(3, 269, 2, 0)],
    "main_tail_16": [(3, 272, 2, 0)],
    "perm_tail_4": [(3, 24, 0, ("perm", 132))],
    "perm_tail_12": [(3, 24, 0, ("perm", 140))],
    "perm_tail_16": [(3, 24, 0, ("perm", 144))],
    "split_over_chips": [(4, 300, 3, 70), (4, 217, 2, 72), (4, 9, 1, 0)],   # 517 main columns, ~350 permutation columns, one height
}


def _wide_spec(orc, name):
    spec = []
    for s in WIDE[name]:
        ints = s[3]
        if isinstance(ints, tuple):
            ints = _n_ints_for_perm_width(orc, s[1], ints[1])
        spec.append((s[0], s[1], s[2], ints))
    return spec


@gpu
@pytest.mark.parametrize("name", list(WIDE))
def test_wide_openings_match_oracle(ctx, orc, name):
    spec = _wide_spec(orc, name)
    chips = _chips(spec, seed=31)
    if len(chips) == 1:
        air = orc.Air(*chips[0][1:])
        if name.startswith("main"):
            assert chips[0][0].shape[0] > 256
        if spec[0][3]:
            assert air.perm_width > 128
        _check_segment(ctx, orc, chips[0])
    _check_chips(ctx, orc, chips)


def test_wide_cases_cross_the_staging_chunks(orc):
    """the widths the cases above are named for"""
    def widths(name):
        chips = _chips(_wide_spec(orc, name), seed=31)
        return [t.shape[0] for t, _, _, _ in chips], [orc.Air(*c[1:]).perm_width for c in chips]
    assert widths("main_517")[0] == [517]
    assert widths("perm_140_interactions")[1][0] > 2 * 128
    for name, tail in (("main_tail_3", 3), ("main_tail_13", 13), ("main_tail_16", 16)):
        assert widths(name)[0][0] % 256 == tail
    for name, tail in (("perm_tail_4", 4), ("perm_tail_12", 12), ("perm_tail_16", 16)):
        assert widths(name)[1][0] % 128 == tail
    m, p = widths("split_over_chips")
    assert sum(m) == 526 and sum(p) > 256


# ---------------------------------------------------------------- 4. edge-valued traces
def _edge_chip(log_n):
    """14 columns: twice each of constant 0, 1, P-1, P-2, alternating 0 / P-1, a P-1 spike at row 0 and one at the last row; AIR
    constraints over all of them and interactions whose multiplicities are the alternating (0 / P-1, a receive of multiplicity -1)
    and spike columns, once negated"""
    from powdr_b200 import machine as M
    n = 1 << log_n
    alt = np.zeros(n, dtype=np.uint32)
    alt[1::2] = P - 1
    first, last = np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.uint32)
    first[0], last[-1] = P - 1, P - 1
    cols = [np.full(n, v, dtype=np.uint32) for v in (0, 1, P - 1, P - 2)] + [alt, first, last]
    trace = np.stack(cols + cols)
    c = ["c%d@%d" % (i, i) for i in range(14)]
    bus_json = [
        {"id": 3, "mult": c[4], "args": [c[2], 17]},
        {"id": 1, "mult": ["-", c[11]], "args": [1, c[3], c[0], c[9], c[10], c[1], [c[12], "+", 65535]]},
        {"id": 6, "mult": c[5], "args": [c[2], c[3], [c[2], "*", c[3]], 1]},
        {"id": 0, "mult": c[6], "args": [c[13], [c[7], "-", [P - 2, "*", c[8]]]]},
        {"id": 2, "mult": c[12], "args": [c[4], c[5], c[6], c[11]]},
    ]
    base = M.synthetic_machine(14, 4, seed=41)
    mach = M.SymbolicMachine(base.constraints, bus_json)
    assert mach.width == 14
    bc, spans = M.compile_constraints(mach)
    return trace, bc, spans, M.compile_bus(mach, 1)


@gpu
@pytest.mark.parametrize("log_n", [9, 10])          # LDE heights 2^10 and 2^11: either side of LEAF_COOP / MERKLE_COOP
def test_edge_valued_trace_matches_oracle(ctx, orc, log_n):
    chip = _edge_chip(log_n)
    _check_segment(ctx, orc, chip)
    _check_segment(ctx, orc, chip, on_device=False)
    _check_chips(ctx, orc, [chip, _edge_chip(log_n - 4)])


def test_edge_valued_trace_oracle_proof_verifies(orc):
    trace, bc, spans, bus = chip = _edge_chip(5)
    assert ((trace[4] == 0) | (trace[4] == P - 1)).all() and {0, P - 1} <= set(trace[4].tolist())
    proof, ys, q, _ = orc.prove(*chip)
    assert orc.verify_segment(bc, spans, 5, 14, proof, ys, q, bus=bus) == 0
