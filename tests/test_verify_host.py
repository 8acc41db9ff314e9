"""The library's host verifier (pb_vk_create, pb_verify_chips, pb_verify_segment) on proofs the oracle writes -- the same proofs as
the GPU prover's, word for word -- without a GPU: it accepts honest proofs, rejects unsatisfying traces and every tampered part with
the same first failure code as the oracle's independent verifier (oracle/verify.c), and refuses what an untrusted proof could get
wrong beyond that (security parameters, shapes, lengths, non-canonical words)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from test_oracle_chips import _chips
from util import P

N_Q, POW = 5, 4


@pytest.fixture(scope="module")
def pb():
    import powdr_b200
    powdr_b200.load_library()
    return powdr_b200


def _keys(pb, chips):
    return [(pb.VerifyingKey(bc, sp, t.shape[0], bus), t.shape[1].bit_length() - 1) for t, bc, sp, bus in chips]


def _zero(chips):
    return [(np.zeros_like(t), bc, sp, bus) for t, bc, sp, bus in chips]


@pytest.mark.parametrize("spec, zero", [
    ([(5, 12, 4, 5), (3, 8, 3, 0), (4, 6, 2, 2)], True),                  # constraints and interactions, padding (all-zero) rows
    ([(6, 12, 0, 7), (4, 9, 0, 0), (4, 14, 0, 5), (3, 10, 0, 3)], False),   # LogUp only, random traces; one chip without anything
    ([(1, 6, 2, 3), (2, 5, 0, 2), (5, 7, 1, 0)], True),                   # 2- and 4-row chips beside a 32-row one
    ([(1, 5, 0, 3), (2, 4, 0, 0)], False),                                # 2- and 4-row chips alone, random
    ([(4, 9, 3, 0), (4, 5, 2, 0)], True),                                 # no interactions anywhere: no permutation commitment
])
def test_oracle_chip_proofs_are_accepted(orc, pb, spec, zero):
    chips = _chips(spec, seed=len(spec))
    if zero:
        chips = _zero(chips)
    proof, cs, ys, q = orc.prove_chips(chips, n_queries=N_Q, pow_bits=POW)
    assert orc.verify_chips(chips, proof, cs, ys, q, check_constraints=True) == 0
    assert pb.verify_chips(_keys(pb, chips), proof, cs, ys, q, n_queries=N_Q, pow_bits=POW) == (0, 0)


@pytest.mark.parametrize("spec", [(1, 6, 2, 3), (2, 9, 0, 4), (5, 10, 3, 0), (6, 12, 4, 6)])
def test_oracle_segment_proofs_are_accepted(orc, pb, spec):
    (trace, bc, spans, bus), = _zero(_chips([spec], seed=7))
    proof, ys, q = orc.prove_segment_q(trace, bc, spans, N_Q, bus=bus, pow_bits=POW)
    (vk, log_n), = _keys(pb, [(trace, bc, spans, bus)])
    assert pb.verify_segment(vk, log_n, proof, ys, q, n_queries=N_Q, pow_bits=POW) == (0, 0)
    bad = dict(proof, perm_width=proof["perm_width"] + 4)          # the key says otherwise: a proof of another shape
    assert pb.verify_segment(vk, log_n, bad, ys, q, n_queries=N_Q, pow_bits=POW) == (pb.capi.PB_ERR_REJECTED, 20)
    assert pb.verify_segment(vk, log_n, bad, ys, q, n_queries=0, pow_bits=POW) == (pb.capi.PB_ERR_INVALID_ARG, 0)   # arguments first
    if not proof["perm_width"]:                                     # no interactions: the cumulative sum is not bound by the transcript
        forged = dict(proof, cumulative_sum=[7, 0, 0, 0])
        assert orc.verify_segment(bc, spans, log_n, trace.shape[0], forged, ys, q, check_constraints=True, bus=bus) == 0
        assert pb.verify_segment(vk, log_n, forged, ys, q, n_queries=N_Q, pow_bits=POW) == (pb.capi.PB_ERR_REJECTED, 20)


def test_unsatisfying_traces_are_rejected_with_the_constraint_identity(orc, pb):
    chips = _chips([(5, 12, 4, 5), (3, 8, 3, 0), (4, 6, 2, 2)], seed=3)
    proof, cs, ys, q = orc.prove_chips(chips, n_queries=N_Q, pow_bits=POW)
    assert orc.verify_chips(chips, proof, cs, ys, q, check_constraints=True) == 16
    assert pb.verify_chips(_keys(pb, chips), proof, cs, ys, q, n_queries=N_Q, pow_bits=POW) == (pb.capi.PB_ERR_REJECTED, 16)


# LogUp-only chips hold the identity for any trace, the constraint chip gets padding rows: every check is reachable
_TAMPER_SPEC = [(5, 10, 0, 4), (3, 7, 0, 3), (4, 9, 3, 0)]


@pytest.fixture(scope="module")
def tamper_case(orc):
    chips = _chips(_TAMPER_SPEC, seed=4)
    chips[2] = (np.zeros_like(chips[2][0]),) + chips[2][1:]
    proof, cs, ys, q = orc.prove_chips(chips, n_queries=N_Q, pow_bits=POW)
    return chips, proof, cs, ys, q


def _layout(orc, chips, proof):
    """offsets into one query's words (include/powdr_b200.h) and into the opened values"""
    widths = [t.shape[0] for t, _, _, _ in chips]
    wps = [orc.Air(bc, sp, bus).perm_width for _, bc, sp, bus in chips]
    lms = [t.shape[1].bit_length() for t, _, _, _ in chips]
    hmax = proof["log_max"]
    hperm = max(lm for lm, wp in zip(lms, wps) if wp)
    wm, wpt, K = sum(widths), sum(wps), len(chips)
    o = {"main_row": 1, "main_path": 1 + wm}
    o["perm_row"] = o["main_path"] + 8 * hmax
    o["perm_path"] = o["perm_row"] + wpt
    o["q_row"] = o["perm_path"] + 8 * hperm
    o["q_path"] = o["q_row"] + 8 * K
    o["fri_pair"] = o["q_path"] + 8 * hmax
    o["fri_path"] = o["fri_pair"] + 8
    n_open = wm + 2 * wpt + 8 * K
    y = {"main": 0, "perm_zeta": wm, "perm_zeta_w": wm + wps[0], "quotient": n_open - 1}
    return o, y


def _bump(v):
    return (int(v) + 1) % P


def _tampers(orc, chips, proof, cs, ys, q):
    """(name, proof, cumsums, ys, queries) with exactly one word changed"""
    o, y = _layout(orc, chips, proof)
    out = []

    def prf(name, key, i, j=None):
        p = {k: [list(r) for r in v] if k in ("fri_roots", "fri_betas", "final_poly") else (list(v) if isinstance(v, list) else v)
             for k, v in proof.items()}
        if j is None:
            p[key][i] = _bump(p[key][i])
        else:
            p[key][i][j] = _bump(p[key][i][j])
        out.append((name, p, cs, ys, q))

    for key in ("main_root", "perm_root", "quotient_root"):
        prf(key, key, 3)
    prf("fri_root_0", "fri_roots", 0, 5)
    prf("fri_root_last", "fri_roots", proof["n_fri_layers"] - 1, 1)
    for key in ("logup_alpha", "logup_beta", "alpha", "zeta", "gamma"):
        prf(key, key, 2)
    prf("fri_beta", "fri_betas", 1, 0)
    prf("final_poly", "final_poly", 1, 3)
    p = dict(proof, pow_witness=(proof["pow_witness"] + 1) % P)
    out.append(("pow_witness", p, cs, ys, q))
    c2 = cs.copy(); c2[1, 2] = _bump(c2[1, 2])
    out.append(("cumsum", proof, c2, ys, q))
    for name, e in y.items():
        y2 = ys.copy(); y2[e, 1] = _bump(y2[e, 1])
        out.append(("ys_" + name, proof, cs, y2, q))
    for name, w in [("r", 0), ("main_row", o["main_row"] + 11), ("main_path", o["main_path"] + 9), ("perm_row", o["perm_row"] + 2),
                    ("perm_path", o["perm_path"]), ("q_row", o["q_row"] + 17), ("q_path", o["q_path"] + 4), ("fri_pair", o["fri_pair"] + 6),
                    ("fri_path", o["fri_path"] + 3), ("last_word", q.shape[1] - 1)]:
        q2 = q.copy(); q2[2, w] = _bump(q2[2, w])
        out.append(("query_" + name, proof, cs, ys, q2))
    return out


def test_tampered_proofs_fail_where_the_oracle_fails(orc, pb, tamper_case):
    chips, proof, cs, ys, q = tamper_case
    keys = _keys(pb, chips)
    assert pb.verify_chips(keys, proof, cs, ys, q, n_queries=N_Q, pow_bits=POW) == (0, 0)
    seen = {}
    for name, p, c, y, qq in _tampers(orc, chips, proof, cs, ys, q):
        want = orc.verify_chips(chips, p, c, y, qq, check_constraints=True)
        rc, why = pb.verify_chips(keys, p, c, y, qq, n_queries=N_Q, pow_bits=POW)
        assert want != 0 and (rc, why) == (pb.capi.PB_ERR_REJECTED, want), (name, want, rc, why)
        seen[name] = why
    # the matrix reaches every check of the transcript and of the queries
    assert {1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 12, 15}.issubset(set(seen.values())), seen
    assert seen["final_poly"] == 15 and seen["query_r"] == 7 and seen["pow_witness"] in (6, 7)


def test_security_parameters_and_shape_come_from_the_verifier(pb, tamper_case):
    chips, proof, cs, ys, q = tamper_case
    keys = _keys(pb, chips)
    rej = pb.capi.PB_ERR_REJECTED
    v = lambda p=proof, **kw: pb.verify_chips(keys, p, cs, ys, q, **dict(dict(n_queries=N_Q, pow_bits=POW), **kw))
    assert v(n_queries=N_Q + 1) == (rej, 21)                     # more queries than the proof has
    assert v(pow_bits=POW + 1) == (rej, 21)                      # more proof of work
    assert v(dict(proof, n_queries=1)) == (rej, 21)              # a proof that claims fewer queries
    assert v(dict(proof, pow_bits=0)) == (rej, 21)
    assert v(dict(proof, n_chips=2)) == (rej, 20)
    assert v(dict(proof, log_max=proof["log_max"] + 1)) == (rej, 20)
    assert v(dict(proof, final_len=1, final_poly=proof["final_poly"][:1])) == (rej, 20)
    # chip 2 has no interactions: a sum in its slot would balance the others' in the caller's bus check, so it must be zero
    c2 = cs.copy(); c2[2] = (-(cs[0].astype(np.int64) + cs[1])) % P
    assert not cs[2].any() and c2[2].any()
    assert pb.verify_chips(keys, proof, c2, ys, q, n_queries=N_Q, pow_bits=POW) == (rej, 20)
    tall = [(keys[0][0], 25)] + keys[1:]
    assert pb.verify_chips(tall, proof, cs, ys, q, n_queries=N_Q, pow_bits=POW) == (rej, 20)


def test_buffer_lengths_must_match_the_chip_shapes(pb, tamper_case):
    chips, proof, cs, ys, q = tamper_case
    keys = _keys(pb, chips)
    bad = pb.capi.PB_ERR_INVALID_ARG
    v = lambda y=ys, qq=q: pb.verify_chips(keys, proof, cs, y, qq, n_queries=N_Q, pow_bits=POW)
    y, qf = ys.ravel(), q.ravel()
    assert v(y=y[:-1]) == (bad, 0) and v(y=np.append(y, 0)) == (bad, 0)
    assert v(qq=qf[:-1]) == (bad, 0) and v(qq=np.append(qf, 0)) == (bad, 0)
    assert pb.verify_chips(keys[:2], proof, cs[:2], ys, q, n_queries=N_Q, pow_bits=POW)[0] == pb.capi.PB_ERR_REJECTED   # n_chips differs
    lib = pb.load_library()
    assert lib.pb_verify_chips(None, C.c_size_t(0), None, None, None, None, C.c_size_t(0), None, C.c_size_t(0), None) == bad


def test_non_canonical_words_are_rejected(pb, tamper_case):
    chips, proof, cs, ys, q = tamper_case
    keys = _keys(pb, chips)
    rej = pb.capi.PB_ERR_REJECTED
    y2 = ys.copy(); y2[4, 0] = P
    assert pb.verify_chips(keys, proof, cs, y2, q, n_queries=N_Q, pow_bits=POW) == (rej, 22)
    q2 = q.copy(); q2[1, 3] = np.uint32(0xffffffff)
    assert pb.verify_chips(keys, proof, cs, ys, q2, n_queries=N_Q, pow_bits=POW) == (rej, 22)
    c2 = cs.copy(); c2[0, 0] += np.uint32(P)
    assert pb.verify_chips(keys, proof, c2, ys, q, n_queries=N_Q, pow_bits=POW) == (rej, 22)
    assert pb.verify_chips(keys, dict(proof, pow_witness=P), cs, ys, q, n_queries=N_Q, pow_bits=POW) == (rej, 22)


def test_other_poseidon2_constants_reject(pb, tamper_case):
    import json
    chips, proof, cs, ys, q = tamper_case
    keys = _keys(pb, chips)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    consts = json.load(open(os.path.join(root, "constants", "poseidon2_babybear_w16.json")))
    ext = np.array(consts["external_initial"] + consts["external_terminal"], dtype=np.uint32)
    inte, diag = [np.array(consts[k], dtype=np.uint32) for k in ("internal", "internal_diag_m1")]
    assert pb.verify_chips(keys, proof, cs, ys, q, n_queries=N_Q, pow_bits=POW, poseidon2=(ext, inte, diag)) == (0, 0)
    inte2 = inte.copy(); inte2[0] = (int(inte2[0]) + 1) % P
    rc, why = pb.verify_chips(keys, proof, cs, ys, q, n_queries=N_Q, pow_bits=POW, poseidon2=(ext, inte2, diag))
    assert rc == pb.capi.PB_ERR_REJECTED and why != 0


# reference-format bytecode: 0 PUSH_APC col, 1 PUSH_CONST c, 2 ADD, 3 SUB, 4 MUL, 5 NEG, 6 INV_OR_ZERO
BAD_CONSTRAINTS = [
    ([9], -4),                            # unknown opcode
    ([0, 3], -4),                         # column >= width (3)
    ([2], -4),                            # stack underflow
    ([0, 0, 0, 1], -4),                   # two values left
    ([0, 0, 0], -4),                      # operand missing
    ([0, 0] * 17 + [2] * 16, -3),         # 17 stack slots
    ([0, 0] * 16 + [2] * 15, 0),          # 16 are fine
]


def _vk_rc(pb, bc, spans, width, bus=None):
    try:
        pb.VerifyingKey(bc, spans, width, bus).free()
        return 0
    except pb.capi.PbError as e:
        return e.code


@pytest.mark.parametrize("bc, code", BAD_CONSTRAINTS)
def test_key_validation_is_the_compile_paths(pb, bc, code):
    lib = pb.load_library()
    spans = [(0, len(bc))]
    assert _vk_rc(pb, bc, spans, 3) == code
    a = np.array(bc, dtype=np.uint32)
    sp = (pb.capi.Span * 1)(pb.capi.Span(0, len(bc)))
    # pb_air_jit_compile_only packs with pb_air_compile's validation; a valid program would go on to NVRTC, so only refusals are compared
    if code:
        assert lib.pb_air_jit_compile_only(a.ctypes.data_as(C.c_void_p), C.c_size_t(a.size), sp, C.c_size_t(1), C.c_uint32(3), None) == code
    assert _vk_rc(pb, bc, [(0, len(bc) + 1)], 3) == -4     # a span past the bytecode


BAD_BUSES = [
    # (interactions [(bus, num_args, args_index_off)], arg spans, bytecode) -> code
    (([(1, 1, 1)], [(0, 2), (2, 2)], [0, 0, 0, 1]), -4),                       # args_index_off + num_args + 1 > spans
    (([(1, 1, 0)], [(0, 2), (2, 2)], [0, 0, 0, 5]), -4),                       # column >= width (4)
    (([(1, 1, 0)], [(0, 11), (11, 2)], [0, 0] * 4 + [4] * 3 + [0, 1]), -2),   # multiplicity of degree 4
    (([(1, 1, 0)], [(0, 3), (3, 2)], [0, 0, 6, 0, 1]), -2),           # OP_INV_OR_ZERO inside an interaction
    (([(1, 1, 0), (2, 1, 2)], [(0, 2), (2, 2), (4, 2), (6, 2)], [0, 0, 0, 1, 0, 2, 0, 3]), 0),
]


@pytest.mark.parametrize("bus, code", BAD_BUSES)
def test_key_interactions_are_validated_and_chunked_as_for_the_prover(pb, bus, code):
    lib = pb.load_library()
    assert _vk_rc(pb, [], [], 4, bus) == code
    if code:
        ints, isp, ibc = bus
        a = np.array(ibc, dtype=np.uint32)
        spn = (pb.capi.Span * len(isp))(*[pb.capi.Span(o, l) for o, l in isp])
        di = (pb.capi.DevInteraction * len(ints))(*[pb.capi.DevInteraction(*t) for t in ints])
        assert lib.pb_air_logup_compile_only(a.ctypes.data_as(C.c_void_p), C.c_size_t(a.size), spn, C.c_size_t(len(isp)), di, C.c_size_t(len(ints)),
                                             C.c_uint32(4), None, None) == code


def test_the_file_passes_with_the_scalar_host_permutation():
    """PB_HOST_P2_SCALAR=1 switches the host permutation to its portable version: the verifier must not depend on which one runs"""
    if os.environ.get("PB_HOST_P2_SCALAR") == "1":
        pytest.skip("already running with the scalar permutation")
    env = dict(os.environ, PB_HOST_P2_SCALAR="1")
    r = subprocess.run([sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "not gpu", os.path.abspath(__file__)],
                       env=env, capture_output=True, text=True, cwd=os.path.dirname(os.path.abspath(__file__)))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
