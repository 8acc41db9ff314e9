"""The proof's byte form (pb_chips_proof_encode, pb_segment_proof_encode, the decoders, pb_verify_proof_bytes) on proofs the oracle
writes -- the GPU prover's proofs, word for word -- without a GPU.  Blobs round-trip; the layout is pinned by a decoder written here
from the header's description and by a golden blob; a tampered blob gets the struct path's verdict; malformed bytes are rejected with
reason 23 before anything past them is read; the C example verifies a file without a device."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from test_oracle_chips import _chips
from test_verify_host import N_Q, POW, _keys, _tampers, _zero, tamper_case  # noqa: F401  (tamper_case: a fixture)
from util import P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "proof_bytes_2chips.bin")
U32 = 0xFFFFFFFF


@pytest.fixture(scope="module")
def pb():
    import powdr_b200
    powdr_b200.load_library()
    return powdr_b200


def _shapes(orc, chips):
    return [(t.shape[1].bit_length() - 1, t.shape[0], orc.Air(bc, sp, bus).perm_width) for t, bc, sp, bus in chips]


def _vks(keys):
    return [vk for vk, _ in keys]


# ---- the layout, restated from the comment in include/powdr_b200.h ----
HEAD = ("magic", "version", "n_chips", "n_queries", "pow_bits", "log_max", "n_fri_layers", "final_len", "reserved")


def _layout_words(chips, n_queries, n_layers, final_len):
    """(n_opened, words_per_query, total words) of a blob with these chips [(log_n, width, perm_width)]"""
    K = len(chips)
    hmax = max(ln + 1 for ln, _, _ in chips)
    hperm = max([ln + 1 for ln, _, wp in chips if wp], default=0)
    wm, wpt = sum(w for _, w, _ in chips), sum(wp for _, _, wp in chips)
    n_open = wm + 2 * wpt + 8 * K
    wpq = 1 + wm + 8 * hmax + (wpt + 8 * hperm if wpt else 0) + 8 * K + 8 * hmax + sum(8 + 8 * (hmax - 1 - i) for i in range(hmax - 1))
    total = 9 + 3 * K + 44 + 12 * n_layers + 4 * final_len + 1 + 4 * K + 4 * n_open + n_queries * wpq
    return n_open, wpq, total


def _py_decode(blob):
    """an independent reader of the format -> (header dict, chips, proof dict, cumulative sums, opened values, queries)"""
    assert len(blob) % 4 == 0
    w = np.frombuffer(blob, dtype="<u4").astype(np.uint32)
    h = dict(zip(HEAD, (int(x) for x in w[:9])))
    K, L, F = h["n_chips"], h["n_fri_layers"], h["final_len"]
    chips = [tuple(int(x) for x in w[9 + 3 * c: 12 + 3 * c]) for c in range(K)]
    pos = [9 + 3 * K]

    def take(n):
        out = w[pos[0]:pos[0] + n]
        pos[0] += n
        return out

    proof = {k: take(8).tolist() for k in ("main_root", "perm_root", "quotient_root")}
    proof.update({k: take(4).tolist() for k in ("logup_alpha", "logup_beta", "alpha", "zeta", "gamma")})
    proof["fri_roots"] = take(8 * L).reshape(L, 8).tolist()
    proof["fri_betas"] = take(4 * L).reshape(L, 4).tolist()
    proof["final_poly"] = take(4 * F).reshape(F, 4).tolist()
    proof["pow_witness"] = int(take(1)[0])
    proof.update(n_fri_layers=L, final_len=F, pow_bits=h["pow_bits"], n_queries=h["n_queries"], n_chips=K, log_max=h["log_max"])
    n_open, wpq, total = _layout_words(chips, h["n_queries"], L, F)
    assert total == w.size
    cs = take(4 * K).reshape(K, 4)
    ys = take(4 * n_open).reshape(n_open, 4)
    q = take(h["n_queries"] * wpq).reshape(h["n_queries"], wpq)
    assert pos[0] == w.size
    return h, chips, proof, cs, ys, q


def _same(got, want):
    gp, gch, gcs, gys, gq = got
    wp, wch, wcs, wys, wq = want
    return gp == wp and list(gch) == list(wch) and np.array_equal(gcs, wcs) and np.array_equal(gys, wys) and np.array_equal(gq, wq)


# ---- round trips ----
@pytest.mark.parametrize("spec, zero", [
    ([(5, 12, 4, 5), (3, 8, 3, 0), (4, 6, 2, 2)], True),                  # the chip mixes of test_verify_host.py
    ([(6, 12, 0, 7), (4, 9, 0, 0), (4, 14, 0, 5), (3, 10, 0, 3)], False),
    ([(1, 6, 2, 3), (2, 5, 0, 2), (5, 7, 1, 0)], True),
    ([(1, 5, 0, 3), (2, 4, 0, 0)], False),
    ([(4, 9, 3, 0), (4, 5, 2, 0)], True),
])
def test_chip_proofs_round_trip_and_verify_from_bytes(orc, pb, spec, zero):
    chips = _chips(spec, seed=len(spec))
    if zero:
        chips = _zero(chips)
    proof, cs, ys, q = orc.prove_chips(chips, n_queries=N_Q, pow_bits=POW)
    shapes = _shapes(orc, chips)
    blob = pb.encode_chips_proof(proof, shapes, cs, ys, q)
    assert _same(pb.decode_proof(blob), (proof, shapes, cs, ys, q))
    h, pchips, pproof, pcs, pys, pq = _py_decode(blob)
    assert (h["magic"], h["version"], h["reserved"]) == (pb.capi.PB_PROOF_MAGIC, 1, 0) and blob[:4] == b"PBPF"
    assert _same((pproof, pchips, pcs, pys, pq), (proof, shapes, cs, ys, q))
    keys = _keys(pb, chips)
    assert pb.verify_proof_bytes(_vks(keys), blob, n_queries=N_Q, pow_bits=POW) == (0, 0)
    assert pb.verify_chips(keys, proof, cs, ys, q, n_queries=N_Q, pow_bits=POW) == (0, 0)


@pytest.mark.parametrize("spec", [(1, 6, 2, 3), (2, 9, 0, 4), (5, 10, 3, 0), (6, 12, 4, 6)])
def test_segment_blob_is_the_one_chip_chips_blob(orc, pb, spec):
    chips = _zero(_chips([spec], seed=7))
    (trace, bc, spans, bus), = chips
    log_n, width = spec[0], trace.shape[0]
    proof, ys, q = orc.prove_segment_q(trace, bc, spans, N_Q, bus=bus, pow_bits=POW)
    blob = pb.encode_segment_proof(proof, log_n, width, ys, q)
    cproof, ccs, cys, cq = orc.prove_chips(chips, n_queries=N_Q, pow_bits=POW)
    assert blob == pb.encode_chips_proof(cproof, _shapes(orc, chips), ccs, cys, cq)
    sp, sln, sw, sys_, sq = pb.decode_proof(blob, segment=True)
    assert (sp, sln, sw) == (proof, log_n, width) and np.array_equal(sys_, ys) and np.array_equal(sq, q)
    (vk, _), = _keys(pb, chips)
    assert pb.verify_proof_bytes([vk], blob, n_queries=N_Q, pow_bits=POW) == (0, 0)


def test_segment_decoder_refuses_other_shapes(orc, pb, tamper_case):
    chips, proof, cs, ys, q = tamper_case
    blob = pb.encode_chips_proof(proof, _shapes(orc, chips), cs, ys, q)
    with pytest.raises(pb.capi.ProofRejected) as e:
        pb.decode_proof(blob, segment=True)             # three chips
    assert e.value.reason == 20
    one = _zero(_chips([(4, 8, 2, 3)], seed=9))
    p1, cs1, ys1, q1 = orc.prove_chips(one, n_queries=N_Q, pow_bits=POW)
    bad = pb.encode_chips_proof(dict(p1, log_max=6), _shapes(orc, one), cs1, ys1, q1)       # a log_max the segment struct cannot hold
    with pytest.raises(pb.capi.ProofRejected) as e:
        pb.decode_proof(bad, segment=True)
    assert e.value.reason == 20
    (vk, _), = _keys(pb, one)
    assert pb.verify_proof_bytes([vk], bad, n_queries=N_Q, pow_bits=POW) == (pb.capi.PB_ERR_REJECTED, 20)


# ---- the golden blob: two chips, the first with interactions ----
def _golden_inputs(orc):
    chips = _zero(_chips([(3, 6, 2, 3), (2, 5, 2, 0)], seed=11))
    return chips, orc.prove_chips(chips, n_queries=3, pow_bits=2)


def test_encoder_reproduces_the_golden_blob(orc, pb):
    """tests/golden/proof_bytes_2chips.bin is the encoder's blob of _golden_inputs, written when the format was fixed: the encoder, the
    oracle's proof and this file's reader must all still agree with it byte for byte"""
    chips, (proof, cs, ys, q) = _golden_inputs(orc)
    blob = pb.encode_chips_proof(proof, _shapes(orc, chips), cs, ys, q)
    with open(GOLDEN, "rb") as f:
        golden = f.read()
    assert blob == golden
    h, pchips, pproof, pcs, pys, pq = _py_decode(golden)
    assert h["n_chips"] == 2 and pchips[0][2] > 0 and pchips[1][2] == 0
    assert _same((pproof, pchips, pcs, pys, pq), (proof, _shapes(orc, chips), cs, ys, q))
    assert pb.verify_proof_bytes(_vks(_keys(pb, chips)), golden, n_queries=3, pow_bits=2) == (0, 0)


# ---- tampering: the blob gets the struct's verdict ----
def test_tampered_blobs_fail_where_the_struct_fails(orc, pb, tamper_case):
    chips, proof, cs, ys, q = tamper_case
    keys, shapes = _keys(pb, chips), _shapes(orc, chips)
    honest = np.frombuffer(pb.encode_chips_proof(proof, shapes, cs, ys, q), dtype="<u4")
    seen = set()
    for name, p, c, y, qq in _tampers(orc, chips, proof, cs, ys, q):
        blob = pb.encode_chips_proof(p, shapes, c, y, qq)
        assert np.count_nonzero(np.frombuffer(blob, dtype="<u4") != honest) == 1, name       # one word of the blob changed
        want = pb.verify_chips(keys, p, c, y, qq, n_queries=N_Q, pow_bits=POW)
        assert want[0] == pb.capi.PB_ERR_REJECTED
        assert pb.verify_proof_bytes(_vks(keys), blob, n_queries=N_Q, pow_bits=POW) == want, name
        seen.add(want[1])
    assert {1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 12, 15}.issubset(seen), seen


def test_security_parameters_shape_and_canonicity_keep_their_codes(orc, pb, tamper_case):
    chips, proof, cs, ys, q = tamper_case
    keys, shapes = _keys(pb, chips), _shapes(orc, chips)
    rej = pb.capi.PB_ERR_REJECTED
    vks = _vks(keys)
    v = lambda blob, **kw: pb.verify_proof_bytes(vks, blob, **dict(dict(n_queries=N_Q, pow_bits=POW), **kw))
    blob = pb.encode_chips_proof(proof, shapes, cs, ys, q)
    assert v(blob, n_queries=N_Q + 1) == (rej, 21) and v(blob, pow_bits=POW + 1) == (rej, 21)
    fewer = pb.encode_chips_proof(dict(proof, n_queries=1), shapes, cs, ys, q[:1])        # a proof that claims fewer queries
    assert v(fewer) == (rej, 21)
    assert v(pb.encode_chips_proof(dict(proof, log_max=proof["log_max"] + 1), shapes, cs, ys, q)) == (rej, 20)
    c2 = cs.copy(); c2[2] = (-(cs[0].astype(np.int64) + cs[1])) % P                      # a sum for the chip without interactions
    assert v(pb.encode_chips_proof(proof, shapes, c2, ys, q)) == (rej, 20)
    y2 = ys.copy(); y2[4, 0] = P
    assert v(pb.encode_chips_proof(proof, shapes, cs, y2, q)) == (rej, 22)
    assert pb.verify_proof_bytes(vks[:2], blob, n_queries=N_Q, pow_bits=POW) == (rej, 20)         # fewer keys than chips
    assert pb.verify_proof_bytes(vks[::-1], blob, n_queries=N_Q, pow_bits=POW) == (rej, 20)       # the keys of other chips


def test_argument_errors(orc, pb, tamper_case):
    chips, proof, cs, ys, q = tamper_case
    keys, shapes = _keys(pb, chips), _shapes(orc, chips)
    lib, bad = pb.load_library(), pb.capi.PB_ERR_INVALID_ARG
    blob = pb.encode_chips_proof(proof, shapes, cs, ys, q)
    for args in [(proof, shapes, cs, ys[:-1], q), (proof, shapes, cs, ys, q[:-1]), (proof, shapes[:2], cs[:2], ys, q),
                 (dict(proof, n_chips=2), shapes, cs, ys, q), (dict(proof, n_fri_layers=33), shapes, cs, ys, q)]:
        with pytest.raises(pb.capi.PbError) as e:
            pb.encode_chips_proof(*args)
        assert e.value.code == bad
    n = C.c_size_t()
    assert lib.pb_chips_proof_encode(None, None, C.c_size_t(0), None, None, C.c_size_t(0), None, C.c_size_t(0), None, C.c_size_t(0), C.byref(n)) == bad
    p = pb.capi.ChipsProof.from_dict(proof)
    arr = (pb.capi.ProofChip * 3)(*[pb.capi.ProofChip(*s) for s in shapes])
    cs_, ys_, q_ = [np.ascontiguousarray(a, dtype=np.uint32) for a in (cs, ys, q)]
    small = C.create_string_buffer(len(blob) - 1)
    assert lib.pb_chips_proof_encode(C.byref(p), arr, C.c_size_t(3), cs_.ctypes.data_as(C.c_void_p), ys_.ctypes.data_as(C.c_void_p), C.c_size_t(ys_.size),
                                     q_.ctypes.data_as(C.c_void_p), C.c_size_t(q_.size), small, C.c_size_t(len(blob) - 1), C.byref(n)) == bad
    prm = pb.capi.VerifyParams(N_Q, POW, None, None, None)
    vks = (C.c_void_p * 3)(*[vk.h.value for vk, _ in keys])
    assert lib.pb_verify_proof_bytes(None, C.c_size_t(3), C.byref(prm), blob, C.c_size_t(len(blob)), None) == bad
    assert lib.pb_verify_proof_bytes(vks, C.c_size_t(0), C.byref(prm), blob, C.c_size_t(len(blob)), None) == bad
    assert lib.pb_verify_proof_bytes(vks, C.c_size_t(3), None, blob, C.c_size_t(len(blob)), None) == bad
    assert lib.pb_verify_proof_bytes(vks, C.c_size_t(3), C.byref(prm), None, C.c_size_t(0), None) == bad
    assert pb.verify_proof_bytes(_vks(keys), blob, n_queries=0, pow_bits=POW) == (bad, 0)      # bad params before the bytes are read
    assert pb.verify_proof_bytes(_vks(keys), b"", n_queries=0, pow_bits=POW) == (bad, 0)
    # the decoder's arrays must have the blob's lengths
    k, nys, nq, why = C.c_size_t(), C.c_size_t(), C.c_size_t(), C.c_int()
    assert lib.pb_proof_bytes_sizes(blob, C.c_size_t(len(blob)), C.byref(k), C.byref(nys), C.byref(nq), C.byref(why)) == 0
    assert (k.value, nys.value, nq.value) == (3, ys.size, q.size)
    out = (pb.capi.ChipsProof(), (pb.capi.ProofChip * 3)(), np.empty(12, np.uint32), np.empty(ys.size, np.uint32), np.empty(q.size, np.uint32))
    dec = lambda kk, ny, nqq: lib.pb_chips_proof_decode(blob, C.c_size_t(len(blob)), C.byref(out[0]), out[1], C.c_size_t(kk), out[2].ctypes.data_as(C.c_void_p),
                                                        out[3].ctypes.data_as(C.c_void_p), C.c_size_t(ny), out[4].ctypes.data_as(C.c_void_p), C.c_size_t(nqq), None)
    assert dec(3, ys.size, q.size) == 0
    assert dec(2, ys.size, q.size) == bad and dec(3, ys.size - 1, q.size) == bad and dec(3, ys.size, q.size - 1) == bad


# ---- malformed bytes ----
def _words(blob):
    return np.frombuffer(blob, dtype="<u4").astype(np.uint32).copy()


def _refit(w, n_queries=None):
    """w with its length made what the header says, where that is computable: then only the field checks can reject it"""
    K = int(w[2])
    if K == 0 or K > 4096 or w.size < 9 + 3 * K:
        return w
    chips = [tuple(int(x) for x in w[9 + 3 * c: 12 + 3 * c]) for c in range(K)]
    if any(not 1 <= ln <= 24 for ln, _, _ in chips) or int(w[6]) > 32 or int(w[7]) > 8:
        return w
    total = _layout_words(chips, int(w[3]), int(w[6]), int(w[7]))[2]
    if total > 1 << 22:
        return w
    return np.concatenate([w, np.zeros(total - w.size, np.uint32)]) if total > w.size else w[:total]


def _expect_malformed(pb, vks, blob):
    rej, lib = pb.capi.PB_ERR_REJECTED, pb.load_library()
    assert pb.verify_proof_bytes(vks, blob, n_queries=N_Q, pow_bits=POW) == (rej, 23)
    k, nys, nq, why = C.c_size_t(), C.c_size_t(), C.c_size_t(), C.c_int()
    assert lib.pb_proof_bytes_sizes(blob, C.c_size_t(len(blob)), C.byref(k), C.byref(nys), C.byref(nq), C.byref(why)) == rej and why.value == 23
    with pytest.raises(pb.capi.ProofRejected) as e:
        pb.decode_proof(blob)
    assert e.value.reason == 23


@pytest.fixture(scope="module")
def small_case(orc, pb):
    chips, (proof, cs, ys, q) = _golden_inputs(orc)
    blob = pb.encode_chips_proof(proof, _shapes(orc, chips), cs, ys, q)
    return _vks(_keys(pb, chips)), blob


def test_truncated_and_extended_blobs_are_malformed(pb, small_case):
    vks, blob = small_case
    for n in range(len(blob) // 4):                      # every word boundary, the empty blob included
        _expect_malformed(pb, vks, blob[:4 * n])
    for cut in (1, 2, 3):
        _expect_malformed(pb, vks, blob[:-cut])
    _expect_malformed(pb, vks, blob + b"\0")
    _expect_malformed(pb, vks, blob + b"\0\0\0\0")
    assert pb.verify_proof_bytes(vks, blob, n_queries=3, pow_bits=2) == (0, 0)


@pytest.mark.parametrize("field, values", [
    (0, [0, 0x46504250 ^ 1, U32]),                                # magic
    (1, [0, 2, U32]),                                             # version
    (8, [1, U32]),                                                # reserved
    (2, [0, 4097, 0x10000, U32]),                                 # n_chips
    (6, [33, U32]),                                               # n_fri_layers
    (7, [9, U32]),                                                # final_len
    (9, [0, 25, U32]),                                            # chip 0 log_n
    (12, [0, 25, U32]),                                           # chip 1 log_n
    (11, [1, 4, 6, 9, 13, U32]),                                  # chip 0 perm_width: not 4 * (chunks + 1)
    (14, [4, 10, 7]),                                             # chip 1 perm_width
])
def test_out_of_range_header_fields_are_malformed(pb, small_case, field, values):
    vks, blob = small_case
    for v in values:
        w = _words(blob)
        w[field] = v
        _expect_malformed(pb, vks, w.astype("<u4").tobytes())
        _expect_malformed(pb, vks, _refit(w).astype("<u4").tobytes())


def test_overflowing_lengths_are_malformed(pb, small_case):
    vks, blob = small_case
    w = _words(blob)
    w[3] = U32                                          # n_queries
    w[10] = U32                                         # chip 0 width: words_per_query above 2^32, times 2^32 queries
    _expect_malformed(pb, vks, w.astype("<u4").tobytes())
    w = _words(blob)
    w[3] = 1 << 31
    w[10] = 1 << 31                                     # 2^31 queries of about 2^31 words: 2^62 words, 2^64 bytes
    _expect_malformed(pb, vks, w.astype("<u4").tobytes())
    # the most chips the format takes, each as wide as possible, queried 2^32 - 1 times
    K = 4096
    head = np.array([0x46504250, 1, K, U32, 2, 25, 24, 2, 0], dtype=np.uint32)
    chips = np.tile(np.array([24, U32, 0xFFFFFFFC], dtype=np.uint32), K)
    _expect_malformed(pb, vks, np.concatenate([head, chips, np.zeros(64, np.uint32)]).astype("<u4").tobytes())
    head[2] = U32                                       # and far more chips than that
    _expect_malformed(pb, vks, np.concatenate([head, chips]).astype("<u4").tobytes())


def test_widths_other_than_the_keys_are_the_proof_shape(orc, pb, small_case):
    vks, blob = small_case
    rej = pb.capi.PB_ERR_REJECTED
    for field, v in [(10, None), (13, None), (11, 4), (14, 8)]:           # widths one more; chip 0's perm_width one chunk more; chip 1 gets one
        w = _words(blob)
        w[field] = int(w[field]) + 1 if v is None else int(w[field]) + v
        w = _refit(w)
        assert pb.verify_proof_bytes(vks, w.astype("<u4").tobytes(), n_queries=3, pow_bits=2) == (rej, 20), field
        pb.decode_proof(w.astype("<u4").tobytes())      # well-formed: only the keys say otherwise


# ---- the C example ----
DEMO_BC = [0, 0, 0, 1, 4, 0, 2, 3, 0, 0, 0, 0, 1, 1, 3, 4, 0, 0, 1, 2, 3, 4]      # a*b - c, a*(a - 1)*(a - 2) (examples/proof_bytes_demo.c)
DEMO_SPANS = [(0, 8), (8, 14)]


def _build_proof_bytes_demo(tmp_path):
    exe = str(tmp_path / "proof_bytes_demo")
    lib_dir = os.path.join(ROOT, "powdr_b200", "_lib")
    subprocess.check_call(["/usr/bin/gcc", "-std=c99", "-O2", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "examples", "proof_bytes_demo.c"), "-L", lib_dir, "-lpowdr_b200", "-Wl,-rpath," + lib_dir, "-o", exe])
    return exe


def test_c_example_verifies_a_file_without_a_device(orc, pb, tmp_path):
    """the example's verify mode reads a blob from a file and never creates a context: an oracle proof of its AIR is accepted, a
    flipped byte is rejected; its prove mode fails loudly without a GPU"""
    exe = _build_proof_bytes_demo(tmp_path)
    rng = np.random.default_rng(5)
    a = rng.integers(0, 3, 64, dtype=np.uint64)
    b = rng.integers(0, P, 64, dtype=np.uint64)
    trace = np.stack([a, b, a * b % P]).astype(np.uint32)
    proof, ys, q = orc.prove_segment_q(trace, DEMO_BC, DEMO_SPANS, 4, pow_bits=16)
    path = tmp_path / "proof.bin"
    path.write_bytes(pb.encode_segment_proof(proof, 6, 3, ys, q))
    r = subprocess.run([exe, "verify", str(path)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and r.stdout.startswith("accepted"), r.stdout + r.stderr
    raw = bytearray(path.read_bytes())
    raw[4 * 14] ^= 1                                     # a word of the main root
    path.write_bytes(bytes(raw))
    r = subprocess.run([exe, "verify", str(path)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 2 and r.stdout.strip().startswith("rejected reason"), r.stdout + r.stderr
    r = subprocess.run([exe, "prove", str(tmp_path / "p2.bin"), "6"], capture_output=True, text=True, timeout=120)
    if r.returncode != 0:
        assert "pb_ctx_create" in r.stderr and "-> -5" in r.stderr, r.stderr
    else:                                                # a GPU is present where this CPU suite runs: the file must then verify
        r = subprocess.run([exe, "verify", str(tmp_path / "p2.bin")], capture_output=True, text=True, timeout=120)
        assert r.returncode == 0, r.stdout + r.stderr
