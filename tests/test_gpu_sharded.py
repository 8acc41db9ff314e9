"""Multi-GPU segment proving (pb_prove_segment_sharded, SURVEY.md §8e) checked on ONE GPU: `world` thread-ranks, each with its
own context, exchange through a barrier + host staging harness (powdr_b200.sharded.ThreadComm) -- the library code path is
the one NCCL drives in bench.py.  The sharded proof must be bit-identical to the single-GPU proof and to the oracle's."""
import numpy as np
import pytest

from util import rand_field

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("log_n,width,world", [(6, 5, 2), (8, 7, 4), (9, 3, 8), (12, 9, 2), (13, 4, 8), (17, 3, 2), (18, 2, 4), (19, 2, 8)])
@pytest.mark.parametrize("shift", [31, 1234567])
def test_lde_shard_is_a_row_block_of_the_lde(ctx, log_n, width, world, shift):
    rng = np.random.default_rng(log_n * 10 + world)
    n = 1 << log_n
    trace = rand_field(rng, (width, n))
    d_in = ctx.to_device(trace)
    d_full = ctx.alloc(4 * width * 2 * n)
    ctx.lde_batch(d_in.ptr, log_n, width, d_full.ptr, 1, shift)
    full = ctx.to_host(d_full, (width, 2 * n))
    ms = 2 * n // world
    d_blk = ctx.alloc(4 * width * ms)
    for blk in range(world):
        ctx.lde_shard(d_in.ptr, log_n, width, world, blk, d_blk.ptr, shift)
        got = ctx.to_host(d_blk, (width, ms))
        assert (got == full[:, blk * ms:(blk + 1) * ms]).all(), blk


def _segment(width, n_constraints, log_n, seed):
    from powdr_b200 import machine as M
    mach = M.synthetic_machine(width, n_constraints, seed=seed)
    bc, spans = M.compile_constraints(mach)
    trace = rand_field(np.random.default_rng(seed), (mach.width, 1 << log_n))
    return bc, spans, trace


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("log_n,width", [(7, 12), (10, 21)])
def test_sharded_proof_equals_single_gpu_and_oracle(ctx, orc, world, log_n, width):
    from powdr_b200.sharded import prove_segment_threads
    bc, spans, trace = _segment(width, 6, log_n, seed=world + log_n)
    air = ctx.air(bc, spans, trace.shape[0])
    d_trace = ctx.to_device(trace)          # keep the buffer alive across the call
    single = ctx.prove_segment(air, d_trace.ptr, log_n, trace.shape[0], on_device=True)
    proofs = prove_segment_threads(world, trace, bc, spans)
    for r, p in enumerate(proofs):
        assert p == single, "rank %d" % r
    assert single == orc.prove_segment(trace, bc, spans)[0]


def test_sharded_proof_mid_size_host_trace(ctx):
    """2^15 rows x 44 columns, 4 ranks, trace shards in host memory; FRI runs sharded for 10 layers before the gather"""
    from powdr_b200.sharded import prove_segment_threads
    bc, spans, trace = _segment(44, 9, 15, seed=3)
    air = ctx.air(bc, spans, trace.shape[0])
    d_trace = ctx.to_device(trace)
    single = ctx.prove_segment(air, d_trace.ptr, 15, trace.shape[0], on_device=True)
    for p in prove_segment_threads(4, trace, bc, spans, on_device=False):
        assert p == single


def test_more_ranks_than_columns(ctx):
    from powdr_b200.sharded import prove_segment_threads
    bc, spans, trace = _segment(5, 3, 8, seed=11)
    air = ctx.air(bc, spans, trace.shape[0])
    d_trace = ctx.to_device(trace)
    single = ctx.prove_segment(air, d_trace.ptr, 8, trace.shape[0], on_device=True)
    assert trace.shape[0] < 8
    for p in prove_segment_threads(8, trace, bc, spans):
        assert p == single


@pytest.mark.parametrize("small", ["2", "5", "24"])
def test_fri_shard_to_replicated_switch_point_does_not_change_the_proof(ctx, monkeypatch, small):
    """PB_SHARD_FRI_SMALL moves the layer at which the FRI codeword is gathered: 2 = fold sharded down to 4 entries per rank
    (a root exchange per layer), 24 = gather immediately"""
    from powdr_b200.sharded import prove_segment_threads
    bc, spans, trace = _segment(10, 4, 11, seed=5)
    air = ctx.air(bc, spans, trace.shape[0])
    d_trace = ctx.to_device(trace)
    single = ctx.prove_segment(air, d_trace.ptr, 11, trace.shape[0], on_device=True)
    monkeypatch.setenv("PB_SHARD_FRI_SMALL", small)
    for p in prove_segment_threads(4, trace, bc, spans):
        assert p == single


@pytest.mark.parametrize("world,log_n,width,n_ints", [(2, 9, 21, 9), (4, 10, 30, 25), (8, 9, 12, 7)])
def test_sharded_logup_segment_equals_single_gpu_and_oracle(ctx, orc, world, log_n, width, n_ints):
    """the LogUp phase on row/column shards (trace transposed to row blocks, permutation trace generated per row block, running sum
    stitched from the gathered block totals, transposed back and LDE'd like the main trace; next-row values of the transition
    constraint fetched from the gathered (S, phi) blocks): every rank's proof equals the single-GPU proof and the oracle's"""
    from powdr_b200 import machine as M
    from powdr_b200.sharded import prove_segment_threads
    base = M.synthetic_machine(width, 4, seed=5)
    mach = M.SymbolicMachine(base.constraints, M.synthetic_bus(base, n_ints, 50 + world, quadratic_every=4))
    bc, spans = M.compile_constraints(mach)
    bus = M.compile_bus(mach, 1)
    trace = rand_field(np.random.default_rng(world), (mach.width, 1 << log_n))
    air = ctx.air(bc, spans, mach.width, bus)
    d = ctx.to_device(trace)
    single = ctx.prove_segment(air, d.ptr, log_n, mach.width, on_device=True)
    assert single == orc.prove(trace, bc, spans, bus, n_queries=8, pow_bits=4)[0]
    for p in prove_segment_threads(world, trace, bc, spans, bus=bus):
        assert p == single
    for p in prove_segment_threads(world, trace, bc, spans, bus=bus, on_device=False):
        assert p == single


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("n_ints", [0, 7])
def test_stage_clocks_of_every_prover_add_up_to_the_total(ctx, world, n_ints):
    """pb_last_stage_ms after pb_prove_segment, pb_prove_chips and every rank of pb_prove_segment_sharded: all 12 slots are set
    (>= 0) and the 11 stages add up to the total"""
    from powdr_b200 import machine as M
    from powdr_b200.sharded import prove_segment_threads
    base = M.synthetic_machine(12, 4, seed=9)
    mach = M.SymbolicMachine(base.constraints, M.synthetic_bus(base, n_ints, 70 + world, quadratic_every=4)) if n_ints else base
    bc, spans = M.compile_constraints(mach)
    bus = M.compile_bus(mach, 1) if n_ints else None
    log_n = 10
    trace = rand_field(np.random.default_rng(world + n_ints), (mach.width, 1 << log_n))
    air = ctx.air(bc, spans, mach.width, bus)
    d = ctx.to_device(trace)
    small = M.synthetic_machine(5, 3, seed=2)
    sbc, sspans = M.compile_constraints(small)
    sair = ctx.air(sbc, sspans, small.width, None)
    sd = ctx.to_device(rand_field(np.random.default_rng(1), (small.width, 1 << 7)))
    clocks = []
    ctx.prove_segment(air, d.ptr, log_n, mach.width, on_device=True)
    clocks.append(("segment", ctx.last_stage_ms()))
    ctx.prove_chips([(air, d.ptr, log_n, mach.width), (sair, sd.ptr, 7, small.width)], want_queries=False)
    clocks.append(("chips", ctx.last_stage_ms()))
    ranks = [None] * world
    prove_segment_threads(world, trace, bc, spans, bus=bus, stage_ms=ranks)
    clocks += [("sharded rank %d" % r, ms) for r, ms in enumerate(ranks)]
    for who, ms in clocks:
        v = list(ms.values())
        assert len(v) == 12 and all(x >= 0 for x in v), (who, ms)
        assert sum(v[:11]) == pytest.approx(v[11], rel=1e-5, abs=1e-3), (who, ms)


@pytest.mark.parametrize("world,log_n,width,n_ints,small", [(2, 9, 21, 9, "14"), (4, 10, 30, 25, "3"), (8, 9, 12, 0, "2"), (4, 13, 9, 4, "6"), (2, 7, 5, 0, "24")])
def test_sharded_query_phase_equals_single_gpu(ctx, orc, monkeypatch, world, log_n, width, n_ints, small):
    """pb_query_segment_sharded: rows and the bottom of every Merkle path from the rank that owns the row block, the top log2(world)
    levels through the gathered subtree roots, FRI layers sharded or replicated depending on the switch point -- every rank ends up
    with exactly the query openings of the single-GPU prover, and the independent verifier accepts them"""
    from powdr_b200 import machine as M
    from powdr_b200.sharded import prove_segment_threads
    base = M.synthetic_machine(width, 4, seed=7)
    mach = M.SymbolicMachine(base.constraints, M.synthetic_bus(base, n_ints, 60 + world, quadratic_every=4)) if n_ints else base
    bc, spans = M.compile_constraints(mach)
    bus = M.compile_bus(mach, 1) if n_ints else None
    trace = rand_field(np.random.default_rng(world + log_n), (mach.width, 1 << log_n))
    air = ctx.air(bc, spans, mach.width, bus)
    d = ctx.to_device(trace)
    single = ctx.prove_segment(air, d.ptr, log_n, mach.width, on_device=True)
    q_single, ys = ctx.query_segment(log_n, mach.width, air.perm_width)
    monkeypatch.setenv("PB_SHARD_FRI_SMALL", small)
    for r, (p, q) in enumerate(prove_segment_threads(world, trace, bc, spans, bus=bus, want_queries=True)):
        assert p == single, "rank %d" % r
        assert (q == q_single).all(), "rank %d" % r
    assert orc.verify_segment(bc, spans, log_n, mach.width, single, ys, q_single, check_constraints=False, bus=bus) == 0
