"""All chips of a segment proved from traces in host memory (pb_prove_chips_host, include/powdr_b200.h): the chips' columns stream over
PCIe in chunks grouped by LDE height, behind the LDE and the leaf hashing (DESIGN.md §3b).  Every proof here is checked word for word
against the oracle (orc_prove_chips) and against pb_prove_chips on device copies of the same traces -- proof, cumulative sums, opened
values, query words -- and must verify (pb_verify_chips) and encode to the device proof's blob.  The chunk schedules are forced small
with PB_PIPE_CHUNK_COLS so that sponge blocks straddle chips, the stream order differs from the chip order, a height group is narrower
than the sponge rate, and the ramped schedule's ragged tail crosses chips."""
import ctypes as C
import hashlib
import json
import os
import sys

import numpy as np
import pytest

from test_gpu_chips import _chips, _gpu_prove
from test_gpu_height_range import _mont
from test_gpu_row_blocks_scale import footprint
from test_proof_bytes_host import _shapes

gpu = pytest.mark.gpu
N_Q, POW = 8, 4                  # the ctx fixture's FRI parameters

# name -> chips (log_n, width, n_constraints, n_interactions[, zero trace]).  So that every proof verifies, a chip is either random
# with interactions only (2 per column: every column is used, so the width is the one asked for) or has constraints and the all-zero
# (padding) trace that satisfies them.
SPECS = {
    "straddle_13_27": [(9, 13, 0, 26), (9, 27, 0, 54)],                                 # a sponge block over the end of one chip and the next
    "interleaved": [(9, 10, 0, 20), (11, 12, 2, 0, True), (9, 14, 0, 28), (11, 9, 0, 18)],   # stream order 1, 3, 0, 2
    "narrow_group": [(10, 20, 0, 40), (8, 5, 0, 10), (6, 11, 1, 3, True)],               # the 2^8 group: one chip of 5 columns
    "ramped_ragged": [(7, 80, 0, 160), (7, 93, 0, 186), (7, 10, 0, 20), (5, 9, 1, 2, True)],   # 183 columns at 2^7: ramp, tail over two chips
}
SEEDS = {name: 300 + i for i, name in enumerate(SPECS)}
BLOCKED_SPEC = [(12, 20, 0, 40), (12, 9, 2, 0, True), (10, 14, 0, 28), (6, 7, 0, 14)]


def chunk_widths(width, chunk_cols):
    """the schedule of one height group (chunk_widths in chips.inl) with PB_PIPE_CHUNK_COLS = chunk_cols"""
    cw = min(width, max(8, chunk_cols // 8 * 8))
    r8 = width % 8
    if width >= 4 * cw + 112:
        mid = width - r8 - 112
        return [8, 16, 32] + [min(cw, mid - k) for k in range(0, mid, cw)] + [32, 16, 8 + r8]
    ws, c0, wk = [], 0, 8
    while c0 < width:
        ws.append(min(wk, width - c0))
        c0 += ws[-1]
        wk = min(cw, 2 * wk)
    return ws


def test_the_specs_reach_the_schedules_they_are_named_for():
    for name, spec in list(SPECS.items()) + [("blocked", BLOCKED_SPEC)]:
        assert [t.shape[0] for t, _, _, _ in _chips(spec, seed=SEEDS.get(name, 41))] == [c[1] for c in spec], name
    for cc in (8, 16):
        # 13 + 27 columns: the second chunk holds the last 5 columns of chip 0 and the first of chip 1
        ws = chunk_widths(40, cc)
        assert ws[0] == 8 < 13 < 8 + ws[1] and sum(ws) == 40
        assert chunk_widths(5, cc) == [5]
        ws = chunk_widths(183, cc)
        assert ws[:3] == [8, 16, 32] and ws[-3:] == [32, 16, 15]
        assert 183 - 15 < 80 + 93 < 183                      # the tail's 15 columns: the last 5 of chip 1, all 10 of chip 2
    assert chunk_widths(150, 8) == [8, 16, 32] + [8] * 4 + [32, 16, 14]     # the one-chip schedule of test_gpu_parity


# ---------------------------------------------------------------- the footprint of K host traces (footprint_bytes, chips.inl)
def footprint_host(chips, lb, h_cut=0):
    """footprint_bytes with host traces: every chip's device copy, and on the resident path one [16][M_h] sponge state per height"""
    words = sum(w << ln for ln, w, _ in chips) + (0 if lb else sum(16 << (ln + 1) for ln in {c[0] for c in chips}))
    return footprint(chips, lb, h_cut) + 4 * words


def choice_host(chips, budget):
    """choose_row_blocks with footprint_host -> (lb, lowest blocked LDE height), (0, None) resident, None when nothing fits"""
    if footprint_host(chips, 0) <= budget:
        return 0, None
    for lb in range(1, 5):
        for h in sorted({c[0] + 1 for c in chips}, reverse=True):
            if h < lb + 4:
                break
            if footprint_host(chips, lb, h) <= budget:
                return lb, h
    return None


def test_the_k_chip_host_footprint_is_the_one_chip_one_at_k_1():
    rng = np.random.default_rng(5)
    for _ in range(20):
        c = [(int(rng.integers(1, 25)), int(rng.integers(1, 3000)), int(rng.choice([0, rng.integers(1, 4000)])))]
        for lb in range(5):
            assert footprint_host(c, lb) == footprint(c, lb, 0, True), (c, lb)


def test_the_blocked_spec_reaches_2_and_4_blocks(orc):
    shp = _shapes(orc, _chips(BLOCKED_SPEC, seed=41))
    for lb in (1, 2):
        assert choice_host(shp, footprint_host(shp, lb, 13)) == (lb, 13)


# ---------------------------------------------------------------- host traces
class HostTraces:
    """the chips' AIRs and their Montgomery traces in host memory: pinned (pb_host_alloc) or pageable numpy arrays"""

    def __init__(self, ctx, chips, pinned=True):
        self.ctx, self.pinned = ctx, pinned
        self.airs = [ctx.air(bc, spans, t.shape[0], bus) for t, bc, spans, bus in chips]
        self.words = [np.ascontiguousarray(_mont(t)) for t, _, _, _ in chips]
        self.ptrs = []
        for m in self.words:
            if pinned:
                p = ctx.host_alloc(m.nbytes)
                C.memmove(p, m.ctypes.data, m.nbytes)
                self.ptrs.append(p)
            else:
                self.ptrs.append(m.ctypes.data)

    def args(self):
        return [(a, p, m.shape[1].bit_length() - 1, m.shape[0]) for a, p, m in zip(self.airs, self.ptrs, self.words)]

    def prove(self):
        return self.ctx.prove_chips(self.args(), on_device=False)

    def overwrite(self):
        for p, m in zip(self.ptrs, self.words):
            C.memset(p, 0x5A, m.nbytes)

    def free(self):
        for a in self.airs:
            a.free()
        if self.pinned:
            for p in self.ptrs:
                self.ctx.host_free(p)


def _prove_host(ctx, chips, pinned=True):
    h = HostTraces(ctx, chips, pinned)
    try:
        return h.prove()
    finally:
        h.free()


def _assert_same(got, exp, what):
    """(proof, cumulative sums, opened values, queries) word for word"""
    assert got[0] == exp[0], what
    assert (got[1] == exp[1]).all(), what
    assert (got[2] == exp[2]).all(), what
    assert got[3].shape == exp[3].shape and (got[3] == exp[3]).all(), what


def _check(ctx, orc, chips, got, n_queries=N_Q, pow_bits=POW, satisfied=True):
    """a host proof = the oracle's = pb_prove_chips on device copies; its blob is the device proof's, and it verifies when the traces
    satisfy their AIRs (satisfied)"""
    from powdr_b200 import VerifyingKey, encode_chips_proof, verify_chips
    _assert_same(got, orc.prove_chips(chips, n_queries=n_queries, pow_bits=pow_bits), "oracle")
    dev = _gpu_prove(ctx, chips)
    _assert_same(got, dev, "device traces")
    shp = _shapes(orc, chips)
    assert encode_chips_proof(got[0], shp, *got[1:]) == encode_chips_proof(dev[0], shp, *dev[1:])
    if not satisfied:
        return
    vks = [VerifyingKey(bc, sp, t.shape[0], bus) for t, bc, sp, bus in chips]
    try:
        keys = [(vk, t.shape[1].bit_length() - 1) for vk, (t, _, _, _) in zip(vks, chips)]
        assert verify_chips(keys, *got, n_queries=n_queries, pow_bits=pow_bits) == (0, 0)
    finally:
        for vk in vks:
            vk.free()


@gpu
@pytest.mark.parametrize("name", ["chips_mixed.json", "chips_tiny.json"])
def test_committed_fixtures_from_host_memory(ctx, orc, name):
    """the multi-chip fixtures (chips_tiny: 2-, 4- and 32-row chips, with and without interactions) from pinned host memory.  Their
    random traces do not satisfy their constraints, so the proofs are checked against the fixture, the oracle and the device proof"""
    golden = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    sys.path.insert(0, golden)
    from make_golden import chips_for
    sha = lambda a: hashlib.sha256(np.ascontiguousarray(a, dtype=np.uint32).tobytes()).hexdigest()
    g = json.load(open(os.path.join(golden, name)))
    chips = chips_for([tuple(x) for x in g["spec"]], g["seed"])
    ctx.set_fri_params(g["n_queries"], g["pow_bits"])
    try:
        got = _prove_host(ctx, chips)
        assert got[0] == g["proof"] and got[1].tolist() == g["cumsums"] and sha(got[2]) == g["ys_sha256"] and sha(got[3]) == g["queries_sha256"]
        _check(ctx, orc, chips, got, g["n_queries"], g["pow_bits"], satisfied=False)
    finally:
        ctx.set_fri_params(N_Q, POW)


@gpu
@pytest.mark.parametrize("chunk_cols", ["8", "16"])
@pytest.mark.parametrize("name", list(SPECS))
def test_forced_chunk_schedules(ctx, orc, monkeypatch, name, chunk_cols):
    chips = _chips(SPECS[name], seed=SEEDS[name])
    monkeypatch.setenv("PB_PIPE_CHUNK_COLS", chunk_cols)
    got = _prove_host(ctx, chips)
    monkeypatch.delenv("PB_PIPE_CHUNK_COLS")
    _check(ctx, orc, chips, got)


@gpu
def test_one_chip_equals_the_segment_prover_from_host_memory(ctx, orc, monkeypatch):
    """pb_prove_chips_host on one chip = pb_prove_segment with a host trace (its K = 1 case) = the oracle"""
    chips = _chips([(8, 43, 3, 6)], seed=12)
    monkeypatch.setenv("PB_PIPE_CHUNK_COLS", "8")
    h = HostTraces(ctx, chips)
    try:
        got = h.prove()
        air, ptr, log_n, w = h.args()[0]
        seg = ctx.prove_segment(air, ptr, log_n, w, on_device=False)
        q1, ys1 = ctx.query_segment(log_n, w, air.perm_width)
    finally:
        h.free()
    proof, cs, ys, q = got
    assert proof["main_root"] == seg["trace_root"] and cs[0].tolist() == seg["cumulative_sum"]
    shared = set(proof) & set(seg)
    assert len(shared) >= 14 and {k: proof[k] for k in shared} == {k: seg[k] for k in shared}
    assert (ys == ys1).all() and (q == q1).all()
    _assert_same(got, orc.prove_chips(chips, n_queries=N_Q, pow_bits=POW), "oracle")


@gpu
def test_pageable_memory_gives_the_pinned_proof(ctx, monkeypatch):
    chips = _chips(SPECS["interleaved"], seed=SEEDS["interleaved"])
    monkeypatch.setenv("PB_PIPE_CHUNK_COLS", "8")
    pinned = _prove_host(ctx, chips, pinned=True)
    pageable = _prove_host(ctx, chips, pinned=False)
    _assert_same(pageable, pinned, "pageable")


@gpu
def test_host_buffers_may_be_overwritten_after_the_call(ctx):
    """the library proves from its own device copy: buffers overwritten right after pb_prove_chips_host returns do not change what
    pb_query_chips answers"""
    from powdr_b200.capi import Chip, ChipsProof
    chips = _chips(SPECS["narrow_group"], seed=SEEDS["narrow_group"])
    h = HostTraces(ctx, chips)
    try:
        ref = h.prove()
        arr = (Chip * len(chips))(*[Chip(a.h.value, p, ln, w) for a, p, ln, w in h.args()])
        proof, cs = ChipsProof(), np.zeros((len(chips), 4), dtype=np.uint32)
        assert ctx.lib.pb_prove_chips_host(ctx.h, arr, C.c_size_t(len(chips)), C.byref(proof), cs.ctypes.data_as(C.c_void_p)) == 0
        h.overwrite()
        ys, q = np.zeros_like(ref[2]), np.zeros_like(ref[3])
        assert ctx.lib.pb_query_chips(ctx.h, q.ctypes.data_as(C.c_void_p), C.c_size_t(q.size), ys.ctypes.data_as(C.c_void_p), C.c_size_t(ys.size)) == 0
    finally:
        h.free()
    _assert_same((proof.as_dict(), cs, ys, q), ref, "after the overwrite")


@gpu
def test_row_blocked_host_proofs_equal_the_resident_one(ctx, orc):
    """budgets from the K-chip host footprint force 2 and 4 row blocks: every chip copied whole, then proved as a device trace"""
    chips = _chips(BLOCKED_SPEC, seed=41)
    shp = _shapes(orc, chips)
    h = HostTraces(ctx, chips)
    try:
        ref = h.prove()
        assert ctx.last_row_blocks() == 0
        for lb in (1, 2):
            ctx.set_memory_budget(footprint_host(shp, lb, 13))
            try:
                got = h.prove()
                assert ctx.last_row_blocks() == lb
            finally:
                ctx.set_memory_budget(0)
            _assert_same(got, ref, lb)
    finally:
        h.free()
    _check(ctx, orc, chips, ref)


@gpu
def test_a_resident_host_proof_allocates_within_its_footprint():
    """the device memory a fresh context holds after a resident host proof is within the K-chip host footprint"""
    import torch
    import powdr_b200
    spec = [(14, 40, 2, 12), (12, 27, 1, 6), (12, 13, 1, 0), (9, 5, 1, 2)]
    chips = _chips(spec, seed=43)
    c = powdr_b200.Context(0)
    try:
        c.set_fri_params(N_Q, POW)
        h = HostTraces(c, chips)
        try:
            shp = [(ln, w, a.perm_width) for (a, _, ln, w) in h.args()]
            c.synchronize()
            before = torch.cuda.mem_get_info(0)[0]
            h.prove()
            c.synchronize()
            after = torch.cuda.mem_get_info(0)[0]
            assert c.last_row_blocks() == 0
        finally:
            h.free()
    finally:
        c.close()
    held = before - after
    assert 0 < held <= footprint_host(shp, 0), (held, footprint_host(shp, 0))


@gpu
def test_argument_checks(ctx):
    """NULL or zero-width chips are refused like pb_prove_chips refuses them, and a refused call leaves no proof to query"""
    from powdr_b200.capi import Chip, ChipsProof
    lib = ctx.lib
    chips = _chips([(5, 12, 4, 5)], seed=4)
    h = HostTraces(ctx, chips)
    try:
        h.prove()
        a, p, ln, w = h.args()[0]
        proof, cs = ChipsProof(), (C.c_uint32 * 4)()
        for bad in (Chip(None, None, 4, 3), Chip(a.h.value, None, ln, w), Chip(a.h.value, p, ln, 0)):
            assert lib.pb_prove_chips_host(ctx.h, (Chip * 1)(bad), C.c_size_t(1), C.byref(proof), cs) == -1
        assert lib.pb_prove_chips_host(ctx.h, (Chip * 1)(Chip(a.h.value, p, ln, w)), C.c_size_t(0), C.byref(proof), cs) == -1
        assert lib.pb_prove_chips_host(ctx.h, None, C.c_size_t(1), C.byref(proof), cs) == -1
        assert lib.pb_query_chips(ctx.h, None, C.c_size_t(0), None, C.c_size_t(0)) == -1
    finally:
        h.free()
