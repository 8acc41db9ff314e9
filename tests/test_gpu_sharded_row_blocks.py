"""Sharded proofs whose rank blocks are proved in row sub-blocks (a memory budget on every rank, include/powdr_b200.h), checked on ONE
GPU with `world` thread-ranks (powdr_b200.sharded.ThreadComm): every rank's proof, cumulative sums, opened values and query words equal
pb_prove_chips + pb_query_chips on the gathered traces and the oracle's, whatever the sub-blocks, the FRI switch point or the queries."""

import numpy as np
import pytest

from test_gpu_chips import _chips
from test_gpu_sharded_chips import _same, _single
from test_sharded_row_blocks_host import choose, footprint_sharded

pytestmark = pytest.mark.gpu

# LDE heights 2^10, 2^9, 2^7: chips with and without interactions; the 2^6-row chip stays whole at every G * B = 16.  The tallest
# chip's permutation trace is wide enough that 2 sub-blocks save memory at every world (they only halve its LDE blocks)
SPEC = [(9, 6, 2, 24), (8, 10, 3, 0), (6, 9, 0, 5)]


def _shapes(ctx, chips):
    out = []
    for t, bc, spans, bus in chips:
        a = ctx.air(bc, spans, t.shape[0], bus)
        out.append((t.shape[1].bit_length() - 1, t.shape[0], a.perm_width))
        a.free()
    return out


def _on_ranks(world, chips, body, devices=None):
    """body(rank, group, ctx, comm, args) on `world` thread-ranks, each with its own context (on devices[rank], default 0), its AIRs and
    its column block of every chip on the device; args as Context.prove_chips_sharded takes them"""
    from powdr_b200.capi import Context
    from powdr_b200.sharded import ThreadComm, _run_ranks, shard_columns

    def run(rank, group):
        c = Context(devices[rank] if devices else 0)
        try:
            c.set_fri_params(8, 4)
            comm = ThreadComm(group, rank, c)
            airs = [c.air(bc, sp, t.shape[0], bus) for t, bc, sp, bus in chips]
            blocks = []
            for t, _, _, _ in chips:
                f, n = shard_columns(t.shape[0], world, rank)
                blocks.append(c.to_device(t[f:f + n]) if n else None)
            args = [(a, b.ptr if b else 0, t.shape[1].bit_length() - 1, t.shape[0]) for a, b, (t, _, _, _) in zip(airs, blocks, chips)]
            out = body(rank, group, c, comm, args)
            assert comm.error is None
            for a in airs:
                a.free()
            return out
        finally:
            c.close()

    return _run_ranks(world, run)


def _budget(shapes, world, lb):
    """the budget of `lb` sub-blocks over every height that can take them, and the path the provers must choose at it"""
    g = world.bit_length() - 1
    cut = min(h for h in {s[0] + 1 for s in shapes} if h >= g + lb + 4)
    budget = footprint_sharded(shapes, world, lb, cut)
    return budget, choose(shapes, world, budget)


@pytest.mark.parametrize("world,lb", [(2, 1), (2, 2), (2, 3), (4, 1), (4, 2), (8, 1)])
def test_blocked_sharded_chips_equal_single_gpu_and_oracle(ctx, orc, world, lb):
    from powdr_b200.sharded import prove_chips_threads
    chips = _chips(SPEC, seed=10 * world + lb)
    shapes = _shapes(ctx, chips)
    budget, path = _budget(shapes, world, lb)
    assert path[0] == lb, path
    single = _single(ctx, chips)
    stats = [None] * world
    for r, got in enumerate(prove_chips_threads(world, chips, stats=stats, budget=budget)):
        assert _same(got, single), "rank %d" % r
        assert stats[r]["log_blocks"] == lb
    proof, cs, ys, q = single
    e_proof, e_cs, e_ys, e_q = orc.prove_chips(chips, n_queries=8, pow_bits=4)
    assert proof == e_proof and (cs == e_cs).all() and (ys == e_ys).all() and (q == e_q).all()
    assert orc.verify_chips(chips, proof, cs, ys, q, check_constraints=False) == 0       # random traces: the transcript and openings
    # the library's host verifier, with the constraint identity: the chips with constraints get all-zero traces, which satisfy them
    from powdr_b200 import VerifyingKey, verify_chips
    zchips = _chips([s + (True,) if s[2] else s for s in SPEC], seed=10 * world + lb)
    keys = [(VerifyingKey(bc, sp, t.shape[0], bus), t.shape[1].bit_length() - 1) for t, bc, sp, bus in zchips]
    stats = [None] * world
    for r, got in enumerate(prove_chips_threads(world, zchips, stats=stats, budget=budget)):
        assert stats[r]["log_blocks"] == lb
        assert verify_chips(keys, *got, n_queries=8, pow_bits=4) == (0, 0), r


@pytest.mark.parametrize("small", ["2", "5", "7", "24"])
def test_fri_switch_points_do_not_change_a_blocked_proof(ctx, monkeypatch, small):
    from powdr_b200.sharded import prove_chips_threads
    chips = _chips(SPEC + [(7, 6, 1, 3)], seed=3)
    budget, path = _budget(_shapes(ctx, chips), 2, 2)
    assert path[0] == 2, path
    single = _single(ctx, chips)
    monkeypatch.setenv("PB_SHARD_FRI_SMALL", small)
    stats = [None] * 2
    for r, got in enumerate(prove_chips_threads(2, chips, budget=budget, stats=stats)):
        assert _same(got, single), "rank %d" % r
        assert stats[r]["log_blocks"] == 2


def _expected_calls(shapes, world, lb, cut, idx, log_max):
    """collectives of a blocked sharded proof and its query phase (DESIGN.md §6) beside those of the resident proof of the same chips:
    per blocked height and sub-step, one all-to-all for its main LDE and, with interactions, one for its permutation LDE, in each of the
    main and permutation commits, the quotient and the reduced opening; in the query phase only the sub-steps that hold a queried row"""
    g = world.bit_length() - 1
    blocked = sorted({s[0] + 1 for s in shapes if s[0] + 1 >= cut and s[0] >= g + lb + 3})
    extra = 0
    for h in blocked:
        lu = any(s[2] for s in shapes if s[0] + 1 == h)
        per_step = 1 + lu
        extra += (1 << lb) * (1 + lu + 2 * per_step)                 # commits, quotient, reduced opening
        hit = {((r >> (log_max - h)) >> (h - g - lb)) & ((1 << lb) - 1) for r in idx}
        extra += len(hit) * per_step                                 # query phase
    resident_main = any(not (s[0] + 1 >= cut and s[0] >= g + lb + 3) for s in shapes)
    resident_perm = any(s[2] and not (s[0] + 1 >= cut and s[0] >= g + lb + 3) for s in shapes)
    return extra - (not resident_main) - (not resident_perm and any(s[2] for s in shapes))


@pytest.mark.parametrize("n_queries", [1, 2, 3])
def test_query_phases_skip_sub_steps_and_count_their_collectives(ctx, n_queries):
    from powdr_b200.sharded import prove_chips_threads
    world, lb = 2, 3
    chips = _chips(SPEC, seed=40 + n_queries)
    shapes = _shapes(ctx, chips)
    budget, path = _budget(shapes, world, lb)
    resident_stats, blocked_stats = [None] * world, [None] * world
    resident = prove_chips_threads(world, chips, fri_params=(n_queries, 2), stats=resident_stats)
    blocked = prove_chips_threads(world, chips, fri_params=(n_queries, 2), stats=blocked_stats, budget=budget)
    for r in range(world):
        assert _same(blocked[r], resident[r]), r
        assert blocked_stats[r]["calls"] == blocked_stats[0]["calls"]
    q = blocked[0][3]
    idx, log_max = [int(v) for v in q[:, 0]], max(s[0] for s in shapes) + 1
    base = sum(resident_stats[0]["calls"].values())
    got = sum(blocked_stats[0]["calls"].values())
    assert got == base + _expected_calls(shapes, world, lb, path[1], idx, log_max), (got, base, path, idx)
    assert blocked_stats[0]["calls"]["all_gather"] == resident_stats[0]["calls"]["all_gather"]


def test_a_budget_reset_to_zero_keeps_todays_collectives(ctx):
    """a blocked proof, then the budget reset to 0 on the same contexts: the resident path with the collectives of a fresh context
    (the counts test_gpu_sharded_chips.py pins), the same proof"""
    from powdr_b200.sharded import prove_chips_threads
    world = 4
    chips = _chips([(9, 6, 2, 24), (9, 10, 2, 5)], seed=2)
    budget, path = _budget(_shapes(ctx, chips), world, 2)
    assert path[0] == 2, path
    fresh = [None] * world
    want = prove_chips_threads(world, chips, stats=fresh)

    def body(rank, group, c, comm, args):
        c.set_memory_budget(budget)
        blocked = c.prove_chips_sharded(args, comm)
        assert c.last_row_blocks() == 2
        before = dict(comm.calls)
        c.set_memory_budget(0)
        resident = c.prove_chips_sharded(args, comm)
        assert c.last_row_blocks() == 0
        return blocked, resident, {k: comm.calls[k] - before[k] for k in before}

    for r, (blocked, resident, calls) in enumerate(_on_ranks(world, chips, body)):
        assert _same(blocked, want[r]) and _same(resident, want[r]), r
        assert calls == fresh[r]["calls"], (r, calls, fresh[r]["calls"])


def test_a_blocked_proof_allocates_within_its_footprint(ctx):
    """the device memory a blocked proof leaves held (its workspaces only grow while it runs, so this is their peak) is within
    pb_footprint_bytes_sharded on every rank: the accounting the choice and its before-any-collective failure rest on"""
    import torch
    world, lb = 2, 2
    chips = _chips([(16, 48, 2, 40), (14, 40, 3, 0), (12, 24, 0, 12)], seed=11)
    shapes = _shapes(ctx, chips)
    budget, path = _budget(shapes, world, lb)
    assert path[0] == lb, path
    used = {}

    def body(rank, group, c, comm, args):
        c.synchronize()
        group.barrier.wait(timeout=120)
        if rank == 0:
            used["before"] = torch.cuda.mem_get_info(0)[0]
        group.barrier.wait(timeout=120)
        c.set_memory_budget(budget)
        c.prove_chips_sharded(args, comm)
        c.synchronize()
        group.barrier.wait(timeout=120)
        if rank == 0:
            used["after"] = torch.cuda.mem_get_info(0)[0]
        group.barrier.wait(timeout=120)
        return c.last_row_blocks()

    assert _on_ranks(world, chips, body) == [lb] * world
    held = used["before"] - used["after"]
    assert 0 < held <= world * budget, (held, world * budget)


def test_nothing_fits_fails_on_every_rank_before_any_collective(ctx):
    from powdr_b200.capi import PbError
    world = 2
    chips = _chips(SPEC, seed=7)
    shapes = _shapes(ctx, chips)
    smallest = min(footprint_sharded(shapes, world, lb) for lb in range(4))
    single = _single(ctx, chips)

    def body(rank, group, c, comm, args):
        c.set_memory_budget(smallest - 1)
        with pytest.raises(PbError) as e:
            c.prove_chips_sharded(args, comm)
        assert e.value.code == 2 and sum(comm.calls.values()) == 0
        c.set_memory_budget(0)
        return c.prove_chips_sharded(args, comm)

    for r, got in enumerate(_on_ranks(world, chips, body)):
        assert _same(got, single), r


def test_sharded_segment_with_host_columns_in_row_blocks(ctx):
    """pb_prove_segment_sharded is the one-chip case: host-resident column shares, blocked at G = 4, B = 2"""
    from powdr_b200 import machine as M
    from powdr_b200.sharded import prove_segment_threads
    from util import rand_field
    base = M.synthetic_machine(11, 4, seed=3)
    mach = M.SymbolicMachine(base.constraints, M.synthetic_bus(base, 24, 31, quadratic_every=4))
    bc, spans = M.compile_constraints(mach)
    bus = M.compile_bus(mach, 1)
    trace = rand_field(np.random.default_rng(5), (mach.width, 1 << 9))
    a = ctx.air(bc, spans, mach.width, bus)
    shapes = [(9, mach.width, a.perm_width)]
    a.free()
    budget = footprint_sharded(shapes, 4, 1, 0, host_trace=True)
    resident = prove_segment_threads(4, trace, bc, spans, bus=bus, on_device=False, want_queries=True)
    stats = [None] * 4
    blocked = prove_segment_threads(4, trace, bc, spans, bus=bus, on_device=False, want_queries=True, stats=stats, budget=budget)
    for r in range(4):
        assert resident[r][0] == blocked[r][0] and (resident[r][1] == blocked[r][1]).all(), r
        assert stats[r]["log_blocks"] == 1


KECCAK = (2022, 187, 1734)          # columns, constraints, interactions of the guest-keccak APC chip (3348 permutation columns)


def test_keccak_shape_at_2p21_rows_on_two_gpus_equals_the_single_gpu_blocked_proof():
    """2^21 x 2022 with 1734 interactions on two GPUs, one thread-rank each, its sub-blocks chosen from an 80 GB-class budget (79 GiB
    less the 8.5 GB column share: B = 8 by the accounting), equals the single-GPU proof at B = 8 word for word.  Needs two 80 GB GPUs"""
    import torch
    if torch.cuda.device_count() < 2 or any(torch.cuda.get_device_properties(d).total_memory < (79 << 30) for d in range(2)):
        pytest.skip("needs two 80 GB-class GPUs: a rank holds 68 GiB beside its 7.9 GiB column share")
    from powdr_b200 import Context
    from powdr_b200 import machine as M
    from util import rand_field
    w, ncons, nints = KECCAK
    base = M.synthetic_machine(w, ncons, seed=21)
    mach = M.SymbolicMachine(base.constraints, M.synthetic_bus(base, nints, seed=22))
    bc, spans = M.compile_constraints(mach)
    bus = M.compile_bus(mach, 1)
    trace = rand_field(np.random.default_rng(21), (mach.width, 1 << 21))
    chips = [(trace, bc, spans, bus)]
    c = Context(0)
    try:
        c.set_fri_params(8, 4)
        air = c.air(bc, spans, mach.width, bus)
        wp = air.perm_width
        d = c.to_device(trace)
        single = c.prove_chips([(air, d.ptr, 21, mach.width)])
        blocks_single = c.last_row_blocks()
        del d
        air.free()
    finally:
        c.close()
    torch.cuda.empty_cache()
    shapes = [(21, mach.width, wp)]
    share = 4 * (-(-mach.width // 2)) * (1 << 21)
    budget = (79 << 30) - share
    path = choose(shapes, 2, budget)
    assert path == (3, 22), path

    def body(rank, group, ctx2, comm, args):
        ctx2.set_memory_budget(budget)
        got = ctx2.prove_chips_sharded(args, comm)
        return got, ctx2.last_row_blocks()

    for r, (got, lb) in enumerate(_on_ranks(2, chips, body, devices=[0, 1])):
        assert lb == 3 and _same(got, single), r
    assert blocks_single >= 1          # one 80 GB GPU proves this shape in row blocks
