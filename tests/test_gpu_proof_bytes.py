"""The byte form of the GPU provers' proofs: the blob of each prover equals the oracle's blob of the same inputs byte for byte and
verifies from its bytes alone -- the single-chip prover with the trace on the device and in host memory, a mixed-height chip set, the
row-blocked path and the sharded prover at G = 2 and 4 on every rank.  The C example proves and writes a file in one process and
verifies it in another.  At the headline shape (2^20 x 2022, 1734 interactions, 100 queries) the blob size, the encode time and the
verification time from bytes next to pb_verify_chips are printed."""
import ctypes as C
import subprocess
import time

import numpy as np
import pytest

from test_gpu_chips import _chips, _gpu_prove
from test_proof_bytes_host import _build_proof_bytes_demo, _shapes
from util import P

pytestmark = pytest.mark.gpu

N_Q, POW = 8, 4          # the ctx fixture's FRI parameters


def _vks(chips):
    from powdr_b200 import VerifyingKey
    return [VerifyingKey(bc, sp, t.shape[0], bus) for t, bc, sp, bus in chips]


def _oracle_blob(orc, chips):
    from powdr_b200 import encode_chips_proof
    proof, cs, ys, q = orc.prove_chips(chips, n_queries=N_Q, pow_bits=POW)
    return encode_chips_proof(proof, _shapes(orc, chips), cs, ys, q)


def _check(orc, chips, got):
    """got: (proof, cumulative sums, opened values, queries) of a GPU prover"""
    from powdr_b200 import encode_chips_proof, verify_proof_bytes
    blob = encode_chips_proof(*got[:1], _shapes(orc, chips), *got[1:])
    assert blob == _oracle_blob(orc, chips)
    assert verify_proof_bytes(_vks(chips), blob, n_queries=N_Q, pow_bits=POW) == (0, 0)


@pytest.mark.parametrize("on_device", [True, False])
def test_segment_blobs_equal_the_oracles(ctx, orc, on_device):
    from powdr_b200 import encode_segment_proof, verify_proof_bytes
    chips = _chips([(9, 14, 4, 6, True)], seed=5)
    (trace, bc, spans, bus), = chips
    width = trace.shape[0]
    air = ctx.air(bc, spans, width, bus)
    if on_device:
        d = ctx.to_device(trace)
        proof = ctx.prove_segment(air, d.ptr, 9, width, on_device=True)
    else:
        host = ((trace.astype(np.uint64) * np.uint64((1 << 32) % P)) % np.uint64(P)).astype(np.uint32)
        proof = ctx.prove_segment(air, host.ctypes.data, 9, width, on_device=False)
    q, ys = ctx.query_segment(9, width, air.perm_width)
    air.free()
    blob = encode_segment_proof(proof, 9, width, ys, q)
    e_proof, e_ys, e_q = orc.prove_segment_q(trace, bc, spans, N_Q, bus=bus, pow_bits=POW)
    assert blob == encode_segment_proof(e_proof, 9, width, e_ys, e_q) == _oracle_blob(orc, chips)
    assert verify_proof_bytes(_vks(chips), blob, n_queries=N_Q, pow_bits=POW) == (0, 0)


def test_mixed_height_chip_blobs_equal_the_oracles(ctx, orc):
    chips = _chips([(6, 12, 0, 7), (4, 9, 2, 0, True), (4, 14, 0, 5), (3, 10, 0, 3), (7, 8, 2, 0, True)], seed=81)
    _check(orc, chips, _gpu_prove(ctx, chips))


def test_row_blocked_blobs_equal_the_oracles(ctx, orc):
    from powdr_b200.capi import footprint_bytes
    chips = _chips([(8, 12, 0, 7), (8, 9, 2, 0, True), (5, 14, 0, 5)], seed=82)
    airs = [ctx.air(bc, sp, t.shape[0], bus) for t, bc, sp, bus in chips]
    bufs = [ctx.to_device(t) for t, _, _, _ in chips]
    arg = [(a, b.ptr, t.shape[1].bit_length() - 1, t.shape[0]) for a, b, (t, _, _, _) in zip(airs, bufs, chips)]
    try:
        for lb in (1, 3):
            ctx.set_memory_budget(footprint_bytes([(t.shape[1].bit_length() - 1, t.shape[0], a.perm_width) for a, (t, _, _, _) in zip(airs, chips)], lb))
            out = ctx.prove_chips(arg)
            assert ctx.last_row_blocks() == lb
            _check(orc, chips, out)
    finally:
        ctx.set_memory_budget(0)
        for a in airs:
            a.free()


@pytest.mark.parametrize("world", [2, 4])
def test_sharded_blobs_equal_the_oracles_on_every_rank(orc, world):
    from powdr_b200.sharded import prove_chips_threads
    chips = _chips([(9, 10, 0, 5), (7, 9, 2, 0, True), (8, 12, 0, 4)], seed=world + 90)
    ranks = prove_chips_threads(world, chips)
    assert len(ranks) == world
    for got in ranks:
        _check(orc, chips, got)


def test_c_example_proves_writes_and_verifies_in_another_process(tmp_path):
    exe = _build_proof_bytes_demo(tmp_path)
    path = str(tmp_path / "proof.bin")
    r = subprocess.run([exe, "prove", path, "10"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.startswith("wrote"), r.stdout + r.stderr
    r = subprocess.run([exe, "verify", path], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.startswith("accepted"), r.stdout + r.stderr


def _median_s(fn, runs=5):
    ts = []
    for _ in range(runs):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), min(ts), max(ts)


def test_headline_blob_size_and_times(ctx):
    """2^20 x 2022 with the 1734-interaction AIR of test_gpu_fullsize.py at 100 queries and 16 proof-of-work bits: the blob verifies,
    and the blob size, the encode time and the verification times (from bytes, and pb_verify_chips on the decoded proof) are printed,
    each the median of 5 runs of the library call on the host"""
    import powdr_b200 as pb
    from powdr_b200 import capi, machine as M
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
    vk = pb.VerifyingKey([], [], w, bus)
    lib = pb.load_library()
    sp = capi.SegmentProof.from_dict(proof)
    y, qq = np.ascontiguousarray(ys), np.ascontiguousarray(q)
    n = C.c_size_t()
    assert lib.pb_segment_proof_encode(C.byref(sp), C.c_size_t(log_n), C.c_size_t(w), y.ctypes.data_as(C.c_void_p), C.c_size_t(y.size),
                                       qq.ctypes.data_as(C.c_void_p), C.c_size_t(qq.size), None, C.c_size_t(0), C.byref(n)) == 0
    out = C.create_string_buffer(n.value)
    enc = lambda: lib.pb_segment_proof_encode(C.byref(sp), C.c_size_t(log_n), C.c_size_t(w), y.ctypes.data_as(C.c_void_p), C.c_size_t(y.size),
                                              qq.ctypes.data_as(C.c_void_p), C.c_size_t(qq.size), out, C.c_size_t(n.value), C.byref(n))
    t_enc = _median_s(enc)
    blob = out.raw[:n.value]
    assert blob == pb.encode_segment_proof(proof, log_n, w, ys, q)
    prm = capi.VerifyParams(100, 16, None, None, None)
    vks = (C.c_void_p * 1)(vk.h.value)
    reason = C.c_int()
    t_bytes = _median_s(lambda: lib.pb_verify_proof_bytes(vks, C.c_size_t(1), C.byref(prm), blob, C.c_size_t(len(blob)), C.byref(reason)))
    assert lib.pb_verify_proof_bytes(vks, C.c_size_t(1), C.byref(prm), blob, C.c_size_t(len(blob)), C.byref(reason)) == 0
    cproof, chips, cs, cys, cq = pb.decode_proof(blob)
    assert chips == [(log_n, w, air.perm_width)]
    cp = capi.ChipsProof.from_dict(cproof)
    vc = (capi.VerifyChip * 1)(capi.VerifyChip(vk.h.value, log_n))
    args = (vc, C.c_size_t(1), C.byref(prm), C.byref(cp), cs.ctypes.data_as(C.c_void_p), cys.ctypes.data_as(C.c_void_p), C.c_size_t(cys.size),
            cq.ctypes.data_as(C.c_void_p), C.c_size_t(cq.size), C.byref(reason))
    t_chips = _median_s(lambda: lib.pb_verify_chips(*args))
    assert lib.pb_verify_chips(*args) == 0
    print("headline blob: %d bytes (%d queries x %d words, %d opened values); encode median %.2f ms (%.2f-%.2f); pb_verify_proof_bytes "
          "median %.1f ms (%.1f-%.1f); pb_verify_chips median %.1f ms (%.1f-%.1f); 5 runs each on the host"
          % (len(blob), q.shape[0], q.shape[1], ys.shape[0], 1e3 * t_enc[0], 1e3 * t_enc[1], 1e3 * t_enc[2], 1e3 * t_bytes[0], 1e3 * t_bytes[1],
             1e3 * t_bytes[2], 1e3 * t_chips[0], 1e3 * t_chips[1], 1e3 * t_chips[2]))
