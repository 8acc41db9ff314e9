"""All chips of a segment under ONE transcript across G ranks (pb_prove_chips_sharded / pb_query_chips_sharded), checked on ONE GPU with
`world` thread-ranks (powdr_b200.sharded.ThreadComm): every rank's proof, cumulative sums, opened values and query openings must equal
pb_prove_chips + pb_query_chips on the gathered traces, and the oracle's."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_chips import _chips
from util import rand_field

pytestmark = pytest.mark.gpu

# the mixes of test_gpu_chips.py::test_chips_proof_matches_oracle_bit_for_bit, heights raised below to at least 2^(g+3)
MIXES = [
    [(6, 12, 0, 7), (4, 9, 2, 0), (4, 14, 0, 5), (3, 10, 0, 3)],
    [(5, 12, 4, 5), (3, 8, 3, 0), (4, 6, 2, 2)],
    [(4, 9, 3, 0), (4, 5, 2, 0)],
    [(3, 10, 0, 3), (7, 8, 2, 0)],
    [(8, 6, 2, 4), (8, 7, 0, 3), (8, 5, 1, 0)],
    [(4, 6, 1, 2), (4, 5, 0, 3), (4, 7, 2, 1), (4, 4, 1, 2), (4, 6, 0, 2)],
    [(5, 3, 1, 0), (6, 10, 0, 4), (5, 2, 1, 2)],            # chips narrower than the world: some ranks hold none of their columns
]


def _raise(spec, world):
    g = world.bit_length() - 1
    up = max(0, g + 3 - min(s[0] for s in spec))
    return [(s[0] + up,) + tuple(s[1:]) for s in spec]


def _single(ctx, chips):
    airs = [ctx.air(bc, spans, t.shape[0], bus) for t, bc, spans, bus in chips]
    bufs = [ctx.to_device(t) for t, _, _, _ in chips]
    out = ctx.prove_chips([(a, b.ptr, t.shape[1].bit_length() - 1, t.shape[0]) for a, b, (t, _, _, _) in zip(airs, bufs, chips)])
    for a in airs:
        a.free()
    return out


def _same(a, b):
    return a[0] == b[0] and (a[1] == b[1]).all() and (a[2] == b[2]).all() and (a[3] is None) == (b[3] is None) and (a[3] is None or (a[3] == b[3]).all())


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("mix", range(len(MIXES)))
def test_sharded_chips_equal_single_gpu_and_oracle(ctx, orc, world, mix):
    from powdr_b200.sharded import prove_chips_threads
    chips = _chips(_raise(MIXES[mix], world), seed=mix)
    single = _single(ctx, chips)
    stats = [None] * world
    for r, got in enumerate(prove_chips_threads(world, chips, stats=stats)):
        assert _same(got, single), "rank %d" % r
    proof, cs, ys, q = single
    e_proof, e_cs, e_ys, e_q = orc.prove_chips(chips, n_queries=8, pow_bits=4)
    assert proof == e_proof and (cs == e_cs).all() and (ys == e_ys).all() and (q == e_q).all()
    assert orc.verify_chips(chips, proof, cs, ys, q, check_constraints=False) == 0
    for r, st in enumerate(stats):          # stage clocks: every slot set, the 11 stages add up to the total
        v = list(st["stage_ms"].values())
        assert len(v) == 12 and all(x >= 0 for x in v), (r, v)
        assert sum(v[:11]) == pytest.approx(v[11], rel=1e-5, abs=1e-3), (r, v)


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("small", ["2", "5", "7", "24"])
def test_fri_switch_point_with_injected_heights_does_not_change_the_proof(ctx, monkeypatch, world, small):
    """LDE heights 2^11, 2^9, 2^7, 2^6, 2^5(world 2): PB_SHARD_FRI_SMALL = 7 at world 2 injects 2^9 and 2^7 on the ranks' blocks and
    gathers 2^6 and 2^5 whole at the switch; 2 injects everything blockwise, 24 gathers everything"""
    from powdr_b200.sharded import prove_chips_threads
    spec = [(10, 9, 2, 3), (8, 7, 0, 4), (6, 6, 1, 2), (5, 5, 2, 0)] + ([(4, 4, 0, 3)] if world == 2 else [])
    chips = _chips(spec, seed=world)
    single = _single(ctx, chips)
    monkeypatch.setenv("PB_SHARD_FRI_SMALL", small)
    for r, got in enumerate(prove_chips_threads(world, chips)):
        assert _same(got, single), "rank %d" % r


@pytest.mark.parametrize("world,n_ints", [(2, 6), (4, 0), (8, 9)])
def test_one_chip_equals_the_sharded_segment_prover(ctx, world, n_ints):
    from powdr_b200 import machine as M
    from powdr_b200.sharded import prove_chips_threads, prove_segment_threads
    base = M.synthetic_machine(11, 4, seed=3)
    mach = M.SymbolicMachine(base.constraints, M.synthetic_bus(base, n_ints, 30 + world, quadratic_every=4)) if n_ints else base
    bc, spans = M.compile_constraints(mach)
    bus = M.compile_bus(mach, 1) if n_ints else None
    trace = rand_field(np.random.default_rng(world), (mach.width, 1 << 9))
    chips = prove_chips_threads(world, [(trace, bc, spans, bus)])
    segs = prove_segment_threads(world, trace, bc, spans, bus=bus, want_queries=True)
    for r, ((proof, cs, ys, q), (seg, q1)) in enumerate(zip(chips, segs)):
        assert proof["main_root"] == seg["trace_root"] and cs[0].tolist() == seg["cumulative_sum"], r
        shared = set(proof) & set(seg)
        assert len(shared) >= 14 and {k: proof[k] for k in shared} == {k: seg[k] for k in shared}, r
        assert (q == q1).all(), r


def _bus_chips(k, log_n, seed):
    return _chips([(log_n, 10, 2, 5)] * k, seed=seed)


def test_collectives_do_not_depend_on_the_number_of_chips(ctx):
    from powdr_b200.sharded import prove_chips_threads, prove_segment_threads
    counts = []
    for k in (2, 6):
        stats = [None] * 4
        prove_chips_threads(4, _bus_chips(k, 7, seed=k), stats=stats)
        assert all(s["calls"] == stats[0]["calls"] for s in stats)
        counts.append(stats[0]["calls"])
    assert counts[0] == counts[1], counts
    # one chip: no more collectives than the sharded segment prover made before it became the one-chip case (2^15 x 44, G = 4:
    # 7 + 1 without interactions, 15 + 1 with 25), and exactly as many as pb_prove_chips_sharded with that chip
    from powdr_b200 import machine as M
    for n_ints, parent in ((0, 8), (25, 16)):
        base = M.synthetic_machine(44, 9, seed=3)
        mach = M.SymbolicMachine(base.constraints, M.synthetic_bus(base, n_ints, 7, quadratic_every=4)) if n_ints else base
        bc, spans = M.compile_constraints(mach)
        bus = M.compile_bus(mach, 1) if n_ints else None
        trace = rand_field(np.random.default_rng(n_ints), (mach.width, 1 << 15))
        seg, one = [None] * 4, [None] * 4
        prove_segment_threads(4, trace, bc, spans, bus=bus, want_queries=True, stats=seg)
        prove_chips_threads(4, [(trace, bc, spans, bus)], stats=one)
        assert sum(seg[0]["calls"].values()) <= parent, seg[0]
        assert seg[0]["calls"] == one[0]["calls"], (seg[0], one[0])


def test_query_and_openings_answer_only_their_own_prover(ctx):
    from powdr_b200.capi import SegmentProof
    from powdr_b200.sharded import ThreadComm, _run_ranks, shard_columns
    chips = _chips([(6, 7, 2, 3), (5, 5, 1, 0)], seed=8)
    world = 2
    out = np.zeros(1 << 18, dtype=np.uint32)
    ptr, cap = out.ctypes.data_as(C.c_void_p), C.c_size_t(out.size)

    def body(rank, group):
        from powdr_b200.capi import Context
        c = Context(0)
        try:
            c.set_fri_params(8, 4)
            lib = c.lib
            comm = ThreadComm(group, rank, c)
            airs = [c.air(bc, sp, t.shape[0], bus) for t, bc, sp, bus in chips]
            blocks = []
            for t, _, _, _ in chips:
                f, n = shard_columns(t.shape[0], world, rank)
                blocks.append(c.to_device(t[f:f + n]))
            args = [(a, b.ptr, t.shape[1].bit_length() - 1, t.shape[0]) for a, b, (t, _, _, _) in zip(airs, blocks, chips)]
            c.prove_chips_sharded(args, comm)
            assert lib.pb_query_chips(c.h, ptr, cap, None, C.c_size_t(0)) == -1
            assert lib.pb_query_segment_sharded(c.h, C.byref(comm.c), ptr, cap) == -1
            assert lib.pb_last_openings(c.h, ptr, cap) == -1
            t0 = chips[0][0]
            assert lib.pb_prove_segment_sharded(c.h, airs[0].h, C.c_void_p(blocks[0].ptr), C.c_size_t(6), C.c_size_t(t0.shape[0]), C.c_uint32(1),
                                                C.byref(comm.c), C.byref(SegmentProof())) == 0
            assert lib.pb_query_chips_sharded(c.h, C.byref(comm.c), ptr, cap, None, C.c_size_t(0)) == -1
            whole = [c.to_device(t) for t, _, _, _ in chips]
            c.prove_chips([(a, w.ptr, ln, wd) for (a, _, ln, wd), w in zip(args, whole)])
            assert lib.pb_query_chips_sharded(c.h, C.byref(comm.c), ptr, cap, None, C.c_size_t(0)) == -1
            c.prove_chips_sharded(args, comm)                     # its own prover makes it answer again
            assert comm.error is None
            for a in airs:
                a.free()
        finally:
            c.close()

    _run_ranks(world, body)


def test_arguments_are_checked_before_any_collective(ctx):
    from powdr_b200.capi import Chip, ChipsProof
    from powdr_b200.sharded import Comm, shard_columns

    class NoCollective(Comm):
        called = 0

        def all_gather(self, send, recv, nbytes):
            NoCollective.called += 1
            raise AssertionError("collective called")

        all_to_all = all_gather

    chips = _chips([(6, 12, 2, 3), (5, 3, 1, 0)], seed=5)          # 12 columns: a non-empty block on each of the 4 ranks
    w0, w1 = chips[0][0].shape[0], chips[1][0].shape[0]
    assert w0 % 4 == 0
    airs = [ctx.air(bc, sp, t.shape[0], bus) for t, bc, sp, bus in chips]
    world = 4
    proof, cs = ChipsProof(), (C.c_uint32 * 8)()
    lib = ctx.lib
    for rank in range(world):
        comm = NoCollective(rank, world)
        blocks = []
        for t, _, _, _ in chips:
            f, n = shard_columns(t.shape[0], world, rank)
            blocks.append(ctx.to_device(t[f:f + n]) if n else None)
        ptrs = [b.ptr if b else None for b in blocks]

        def call(specs, k=2, cm=comm):
            arr = (Chip * max(1, k))(*[Chip(*s) for s in specs[:max(1, k)]])
            return lib.pb_prove_chips_sharded(ctx.h, arr, C.c_size_t(k), C.byref(cm.c) if cm else None, C.byref(proof), cs)

        good = [(airs[0].h.value, ptrs[0], 6, w0), (airs[1].h.value, ptrs[1], 5, w1)]
        assert call(good, cm=None) == -1                                                       # NULL comm
        assert call(good, k=0) == -1                                                           # no chips
        assert call([good[0], (None, ptrs[1], 5, w1)]) == -1                                   # NULL air
        assert call([good[0], (airs[1].h.value, ptrs[1], 5, w1 + 1)]) == -1                   # width mismatch
        assert call([good[0], (airs[1].h.value, ptrs[1], 4, w1)]) == -2                       # 2^4 rows < 2^(g+3) on 4 ranks
        assert call([(airs[0].h.value, None, 6, w0), good[1]]) == -1                           # NULL trace for a non-empty block
        bad_world = NoCollective(rank, 3)
        assert call(good, cm=bad_world) == -2
    assert NoCollective.called == 0
    for a in airs:
        a.free()


def test_sharded_chips_at_scale_verify(ctx, orc):
    """G = 4, 2^14 / 2^12 / 2^9 rows with a few hundred interactions: every rank equals the single-GPU proof, and the independent
    verifier accepts it with the constraint identity"""
    from powdr_b200.sharded import prove_chips_threads
    chips = _chips([(14, 64, 0, 120), (12, 40, 0, 60), (9, 30, 3, 0, True), (12, 24, 0, 33)], seed=9)
    single = _single(ctx, chips)
    for r, got in enumerate(prove_chips_threads(4, chips)):
        assert _same(got, single), "rank %d" % r
    assert orc.verify_chips(chips, *single, check_constraints=True) == 0
