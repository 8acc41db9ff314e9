"""CPU tests of the multi-chip segment proof under ONE transcript (oracle/prove.c: orc_prove_chips, oracle/verify.c: orc_verify_chips):
mixed-height MMCS commitments, shared challenges, per-height injection of the reduced openings into one FRI instance."""
import numpy as np
import pytest

from util import P, rand_field


def _chips(spec, seed=0):
    """spec: list of (log_n, width, n_constraints, n_interactions)"""
    from powdr_b200 import machine as M
    rng = np.random.default_rng(seed)
    out = []
    for i, (log_n, width, ncons, nints) in enumerate(spec):
        base = M.synthetic_machine(width, ncons, seed=100 + i) if ncons else None
        bus_json = M.synthetic_bus(width, nints, seed=200 + i, quadratic_every=5) if nints else []
        mach = M.SymbolicMachine(base.constraints if base else [], bus_json)
        bc, spans = M.compile_constraints(mach)
        bus = M.compile_bus(mach, 1) if nints else None
        trace = rand_field(rng, (mach.width, 1 << log_n))
        out.append((trace, bc, spans, bus))
    return out


def test_mixed_heights_with_and_without_interactions_verify(orc):
    # heights 2^6, 2^4, 2^4, 2^3; the second chip has no interactions, the tallest has no constraints of its own
    chips = _chips([(6, 12, 0, 7), (4, 9, 0, 0), (4, 14, 0, 5), (3, 10, 0, 3)], seed=1)
    proof, cs, ys, q = orc.prove_chips(chips, n_queries=6, pow_bits=5)
    assert proof["n_chips"] == 4 and proof["log_max"] == 7 and proof["n_fri_layers"] == 6
    assert proof["final_poly"][0] == proof["final_poly"][1]
    # interaction-only / empty AIRs: every chip's identity at zeta holds for any trace
    assert orc.verify_chips(chips, proof, cs, ys, q, check_constraints=True) == 0
    if orc.fast_available():
        p2, cs2, ys2, q2 = orc.prove_chips(chips, n_queries=6, pow_bits=5, fast=True)
        assert p2 == proof and (cs2 == cs).all() and (ys2 == ys).all() and (q2 == q).all()


def test_one_chip_proofs_reproduce_the_single_segment_fixture(orc):
    """tests/golden/segment_shapes.json pins single-segment proofs of 2-, 4- and 32-row traces (AIRs with constraints and
    interactions, constraints only, interactions only) as a dedicated single-chip prover wrote them; the one-chip proof must be
    the same proof, opened values and query words, in slow and in fast mode"""
    import hashlib
    import json
    import os
    import sys
    golden = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    sys.path.insert(0, golden)
    from make_golden import chips_for
    sha = lambda a: hashlib.sha256(np.ascontiguousarray(a, dtype=np.uint32).tobytes()).hexdigest()
    g = json.load(open(os.path.join(golden, "segment_shapes.json")))
    assert len(g["cases"]) == 9
    for case in g["cases"]:
        trace, bc, spans, bus = chips_for([case["spec"]], g["seed"])[0]
        for fast in ([False, True] if orc.fast_available() else [False]):
            proof, ys, q, _ = orc.prove(trace, bc, spans, bus, n_queries=g["n_queries"], pow_bits=g["pow_bits"], fast=fast)
            assert proof == case["proof"] and sha(ys) == case["ys_sha256"] and sha(q) == case["queries_sha256"], (case["spec"], fast)
        assert orc.verify_segment(bc, spans, case["spec"][0], trace.shape[0], proof, ys, q, bus=bus) == 0


def test_satisfying_and_unsatisfying_traces(orc):
    from powdr_b200 import machine as M
    chips = _chips([(5, 12, 4, 5), (3, 8, 3, 0), (4, 6, 2, 2)], seed=3)
    zero = [(np.zeros_like(t), bc, sp, bus) for t, bc, sp, bus in chips]           # padding rows satisfy the guarded constraints
    proof, cs, ys, q = orc.prove_chips(zero, n_queries=5, pow_bits=4)
    assert orc.verify_chips(zero, proof, cs, ys, q, check_constraints=True) == 0
    proof, cs, ys, q = orc.prove_chips(chips, n_queries=5, pow_bits=4)            # random traces: PCS part fine, identity fails
    assert orc.verify_chips(chips, proof, cs, ys, q, check_constraints=False) == 0
    assert orc.verify_chips(chips, proof, cs, ys, q, check_constraints=True) == 16


def test_tampering_is_rejected(orc):
    chips = _chips([(5, 10, 0, 4), (3, 7, 0, 3), (4, 9, 0, 0)], seed=4)
    proof, cs, ys, q = orc.prove_chips(chips, n_queries=5, pow_bits=4)
    v = lambda p=proof, c=cs, y=ys, qq=q: orc.verify_chips(chips, p, c, y, qq, True)
    assert v() == 0
    c2 = cs.copy(); c2[1, 0] = (int(c2[1, 0]) + 1) % P
    assert v(c=c2) == 2                                   # every chip's cumulative sum is bound by the transcript
    y2 = ys.copy(); y2[-3, 2] = (int(y2[-3, 2]) + 1) % P
    assert v(y=y2) == 4
    q2 = q.copy(); q2[0, 1 + 10 + 2] ^= 1                 # a word of the SECOND chip's main row (injected two levels up the tree)
    assert v(qq=q2) == 8
    total_main = sum(t.shape[0] for t, _, _, _ in chips)
    q3 = q.copy(); q3[1, 1 + total_main + 8 * 6 + 1] ^= 1  # permutation rows
    assert v(qq=q3) == 9
    p2 = dict(proof); p2["final_poly"] = [proof["final_poly"][0], [(proof["final_poly"][1][0] + 1) % P] + proof["final_poly"][1][1:]]
    assert v(p2) == 15


def test_random_chip_mixes_verify_and_bind_every_opened_value(orc):
    """hypothesis: 2-4 chips of random heights / widths / interaction counts under one transcript -- the verifier accepts the honest
    proof and rejects it after ANY single opened value, cumulative sum or query word is changed"""
    from hypothesis import given, settings, strategies as st

    chip = st.tuples(st.integers(3, 6), st.integers(4, 12), st.integers(0, 3), st.integers(0, 4))

    @settings(max_examples=8, deadline=None)
    @given(st.lists(chip, min_size=2, max_size=4), st.integers(0, 2**31), st.data())
    def run(spec, seed, data):
        spec = [(ln, w, nc if (nc or ni) else 1, ni) for ln, w, nc, ni in spec]       # every chip needs at least one column user
        chips = _chips(spec, seed=seed)
        proof, cs, ys, q = orc.prove_chips(chips, n_queries=3, pow_bits=2)
        assert orc.verify_chips(chips, proof, cs, ys, q, check_constraints=False) == 0
        y2 = ys.copy()
        i, l = data.draw(st.integers(0, ys.shape[0] - 1)), data.draw(st.integers(0, 3))
        y2[i, l] = (int(y2[i, l]) + 1) % P
        assert orc.verify_chips(chips, proof, cs, y2, q, check_constraints=False) != 0
        q2 = q.copy()
        qi, w = data.draw(st.integers(0, q.shape[0] - 1)), data.draw(st.integers(1, q.shape[1] - 1))
        q2[qi, w] = (int(q2[qi, w]) + 1) % P
        assert orc.verify_chips(chips, proof, cs, ys, q2, check_constraints=False) != 0
        if cs.any():
            c2 = cs.copy()
            k = int(np.flatnonzero(cs.any(axis=1))[0])
            c2[k, 0] = (int(c2[k, 0]) + 1) % P
            assert orc.verify_chips(chips, proof, c2, ys, q, check_constraints=False) != 0

    run()


def test_committed_fixtures_are_reproduced(orc):
    """tests/golden/segment_2p8_w12.json, segment_logup_2p7.json, chips_mixed.json and chips_tiny.json (written by
    tests/golden/make_golden.py): regression pins of transcript v2 without and with the LogUp phase and of the multi-chip
    transcript -- proof fields exactly, opened values / query openings by digest"""
    import hashlib
    import json
    import os
    import sys
    from powdr_b200 import machine as M
    golden = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    sys.path.insert(0, golden)
    from make_golden import chips_for
    sha = lambda a: hashlib.sha256(np.ascontiguousarray(a, dtype=np.uint32).tobytes()).hexdigest()
    g = json.load(open(os.path.join(golden, "segment_2p8_w12.json")))
    mach = M.synthetic_machine(g["width"], g["n_constraints"], seed=g["seed"])
    bc, spans = M.compile_constraints(mach)
    trace = rand_field(np.random.default_rng(g["trace_seed"]), (mach.width, 1 << g["log_n"]))
    for fast in ([False, True] if orc.fast_available() else [False]):
        assert orc.prove_segment(trace, bc, spans, fast=fast)[0] == g["proof"]
    g = json.load(open(os.path.join(golden, "segment_logup_2p7.json")))
    base = M.synthetic_machine(g["width"], g["n_constraints"], seed=g["seed"])
    mach = M.SymbolicMachine(base.constraints, M.synthetic_bus(base, g["n_interactions"], g["bus_seed"], g["quadratic_every"]))
    bc, spans = M.compile_constraints(mach)
    trace = rand_field(np.random.default_rng(g["trace_seed"]), (mach.width, 1 << g["log_n"]))
    for fast in ([False, True] if orc.fast_available() else [False]):
        proof, ys, q, _ = orc.prove(trace, bc, spans, M.compile_bus(mach, 1), n_queries=g["n_queries"], pow_bits=g["pow_bits"], fast=fast)
        assert proof == g["proof"] and sha(ys) == g["ys_sha256"] and sha(q) == g["queries_sha256"]
    for name in ("chips_mixed.json", "chips_tiny.json"):          # chips_tiny: 2-, 4- and 32-row chips, the bottom of the height range
        g = json.load(open(os.path.join(golden, name)))
        chips = chips_for([tuple(x) for x in g["spec"]], g["seed"])
        for fast in ([False, True] if orc.fast_available() else [False]):
            proof, cs, ys, q = orc.prove_chips(chips, n_queries=g["n_queries"], pow_bits=g["pow_bits"], fast=fast)
            assert proof == g["proof"] and cs.tolist() == g["cumsums"] and sha(ys) == g["ys_sha256"] and sha(q) == g["queries_sha256"], name
        assert orc.verify_chips(chips, proof, cs, ys, q, check_constraints=False) == 0
