"""The row-blocked path of the single-GPU provers (DESIGN.md §3c) at the heights it exists for, word for word:

  1. pb_lde_shard at 4 and 16 blocks (the fold of 2 and 8 coefficients per output, block shifts over 2 and 8 sub-blocks per coset) at
     every size where the block's forward pass changes geometry, against the oracle LDE;
  2. one-chip segments of 2^12 to 2^20 rows in 2, 4, 8 and 16 row blocks against the resident proof of the same context, and the
     resident proof against the oracle (its AVX-512 arm; the sampled checks of test_gpu_height_range without it);
  3. a tall mix of six chips at every (row blocks, lowest blocked height) pair choose_row_blocks can pick;
  4. query phases that skip blocks: 1 to 3 queries over 16 blocks of two blocked heights, two of them in one block;
  5. more than 64 block twiddle sets in one proof (FIFO eviction of get_twiddles in the middle of a proof), twice;
  6. blocked against sharded: the thread-rank sharded prover at 4 and 16 ranks on one GPU, and the 2^21 x 2022 keccak shape in 8 and
     16 blocks on one GPU against 4 GPUs.

B is forced with a memory budget.  The expected choice of the prover is derived here from a restatement of pb_footprint_bytes that
also takes the lowest blocked height (the library exports only "every height that can be blocked"), checked against the library
at the heights the two share."""
import ctypes as C
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from test_gpu_chips import _chips
from test_gpu_height_range import _mont, _n_ints_for_perm_width, _sampled_checks
from test_gpu_lde import SENTINEL, LdeRefs, assert_lde_equal, geom_width, mont, quotient_shift, random_shift
from util import P

gpu = pytest.mark.gpu


# ---------------------------------------------------------------- the footprint and the choice of the path (chips.inl)
FOOTPRINT_SMS, FOOTPRINT_RESERVE = 132, 64 << 20


def footprint(chips, lb, h_cut=0, host_trace=False):
    """footprint_bytes of chips.inl: chips [(log_n, width, perm_width)], the LDE heights >= 2^h_cut with log_n >= lb + 3 in 2^lb blocks"""
    words = n_max = n_lu = m_perm = raw = s = scratch = 0
    for log_n, width, wp in chips:
        N = 1 << log_n
        M = 2 * N
        bl = lb > 0 and log_n + 1 >= h_cut and log_n >= lb + 3
        Ms = M >> (lb if bl else 0)
        words += width * N + width * Ms if bl else width * M
        words += wp * N + wp * Ms
        words += 8 * N + 8 * M
        n_max = max(n_max, N)
        if wp:
            n_lu, m_perm = max(n_lu, N), max(m_perm, M)
            raw = max(raw, 4 * (M + Ms) if bl else 4 * M)
            s = max(s, 8 * M if bl else 4 * M)
        elif bl:
            raw = max(raw, 4 * Ms)
        scratch = max(scratch, 3 * min(max(width, wp, 8) * N, max(N, (16 * FOOTPRINT_SMS) << 15)))
    m_max = 2 * n_max
    words += raw + s + 4 * n_lu + scratch
    words += 16 * m_max * 2 + 16 * m_perm + 8 * m_max
    words += 8 * n_max + 4 * m_max + 4 * n_max
    words += 8 * m_max + 16 * m_max + 4 * m_max
    words += 32 * n_max
    if host_trace:
        words += chips[0][1] * n_max + (0 if lb else 16 * m_max)
    return 4 * words + FOOTPRINT_RESERVE


def choice(chips, budget, host_trace=False):
    """choose_row_blocks: resident (0, None) when the footprint fits; else the fewest blocks 2^lb and, at that lb, the fewest blocked
    heights (tallest first) that fit -> (lb, lowest blocked LDE height); None when nothing fits"""
    if footprint(chips, 0, 0, host_trace) <= budget:
        return 0, None
    heights = sorted({c[0] + 1 for c in chips}, reverse=True)
    for lb in range(1, 5):
        for h in heights:
            if h < lb + 4:
                break
            if footprint(chips, lb, h, host_trace) <= budget:
                return lb, h
    return None


def shapes(orc, chips):
    return [(t.shape[1].bit_length() - 1, t.shape[0], orc.Air(bc, spans, bus).perm_width) for t, bc, spans, bus in chips]


def budget_for(shp, lb, h, host_trace=False):
    """a budget at which choose_row_blocks picks (lb, h), asserted"""
    b = footprint(shp, lb, h, host_trace)
    assert choice(shp, b, host_trace) == (lb, h), (lb, h, choice(shp, b, host_trace))
    return b


def test_footprint_restatement_equals_the_library():
    from powdr_b200.capi import footprint_bytes
    rng = np.random.default_rng(3)
    sets = [[(21, 2022, 3348)], [(12, 64, 40), (6, 64, 40)], [(20, 8, 0), (18, 10, 24), (7, 5, 3), (2, 4, 0)]]
    sets += [[(int(rng.integers(1, 25)), int(rng.integers(1, 3000)), int(rng.choice([0, rng.integers(1, 4000)]))) for _ in range(k)]
             for k in (1, 2, 3, 6) for _ in range(8)]
    for shp in sets:
        for lb in range(5):
            assert footprint(shp, lb) == footprint_bytes(shp, lb), (shp, lb)


# ---------------------------------------------------------------- 1. the 16-block LDE (pb_lde_shard) against the oracle
@pytest.fixture(scope="module")
def refs(orc):
    return LdeRefs(orc)


SHARD_SIZES = ["min", 11, 12, 16, 20, 24]       # min: log_n = g + 3, the shortest height the blocks allow


@gpu
@pytest.mark.parametrize("shift_kind", ["31", "quotient", "random"])
@pytest.mark.parametrize("world", [4, 16])
@pytest.mark.parametrize("size", SHARD_SIZES)
def test_lde_shard_at_4_and_16_blocks_matches_oracle(ctx, refs, size, world, shift_kind):
    """block b = rows [b Ms, (b + 1) Ms) of the 2-coset LDE, Ms = 2N / world: the fold of G1 = world / 2 coefficients per output with
    lambda of the block's shift, then a forward pass of 2^(n + 1 - g) rows; the input comes back unchanged"""
    g = world.bit_length() - 1
    log_n = g + 3 if size == "min" else size
    shift = {"31": 31, "quotient": quotient_shift(log_n), "random": random_shift(log_n)}[shift_kind]
    width = geom_width(log_n)
    plan = [(log_n, log_n, width, 1, s) for s in (31, quotient_shift(log_n), random_shift(log_n))]
    exp = refs.get((log_n, log_n, width, 1, shift), plan)
    words = mont(refs.trace(log_n, log_n, width))
    ms = (2 << log_n) // world
    d_in = ctx.to_device(words, monty=False)
    d_blk = ctx.alloc(4 * width * ms)
    sentinel = np.full(width * ms, SENTINEL, dtype=np.uint32)
    try:
        for blk in range(world):
            d_blk.upload(sentinel)
            ctx.lde_shard(d_in.ptr, log_n, width, world, blk, d_blk.ptr, shift)
            got = d_blk.download((width, ms))
            assert_lde_equal(got, exp[:, blk * ms:(blk + 1) * ms], log_n, 1, row0=blk * ms, what="block %d of %d" % (blk, world))
        assert (d_in.download(words.shape) == words).all(), "pb_lde_shard changed its input"
    finally:
        d_in.free()
        d_blk.free()


# ---------------------------------------------------------------- proofs
def _prove_chips(ctx, airs, bufs, chips):
    return ctx.prove_chips([(a, b.ptr, t.shape[1].bit_length() - 1, t.shape[0]) for a, b, (t, _, _, _) in zip(airs, bufs, chips)])


def _assert_same(got, exp, what):
    """(proof, cumulative sums, opened values, queries) word for word"""
    assert got[0] == exp[0], what
    assert (got[1] == exp[1]).all() and (got[2] == exp[2]).all(), what
    assert got[3].shape == exp[3].shape and (got[3] == exp[3]).all(), what


class ChipSet:
    """chips compiled and uploaded in one context; prove(budget) -> the tuple of prove_chips and the row blocks chosen"""

    def __init__(self, ctx, chips):
        self.ctx, self.chips = ctx, chips
        self.airs = [ctx.air(bc, spans, t.shape[0], bus) for t, bc, spans, bus in chips]
        self.bufs = [ctx.to_device(t) for t, _, _, _ in chips]

    def prove(self, budget):
        self.ctx.set_memory_budget(budget)
        try:
            out = _prove_chips(self.ctx, self.airs, self.bufs, self.chips)
            return out, self.ctx.last_row_blocks()
        finally:
            self.ctx.set_memory_budget(0)

    def free(self):
        for a in self.airs:
            a.free()
        for b in self.bufs:
            b.free()


# ---------------------------------------------------------------- 2. one-chip segments at 2^12 to 2^20 rows
SEGMENTS = {                 # name -> ((log_n, width, n_constraints, n_interactions), trace on the device)
    "2p12": ((12, 10, 3, 5), True),
    "2p14_perm_140": ((14, 24, 2, ("perm", 140)), True),       # wider than one gamma staging chunk (128 columns at two points)
    "2p16": ((16, 12, 3, 8), True),
    "2p18_host_trace": ((18, 12, 3, 8), False),
    "2p20": ((20, 10, 2, 10), True),
}
TALL_MIX = [(20, 8, 2, 6), (18, 10, 0, 8), (18, 6, 3, 0), (14, 12, 2, 5), (7, 9, 1, 3), (2, 5, 1, 2)]


def _segment_chip(orc, name):
    (log_n, width, ncons, nints), _ = SEGMENTS[name]
    if isinstance(nints, tuple):
        nints = _n_ints_for_perm_width(orc, width, nints[1])
    return _chips([(log_n, width, ncons, nints)], seed=log_n + 60)[0]


class ScaleRefs:
    """the chips of 2. and 3. and, with the AVX-512 oracle arm, its proofs of them, started together on first use and computed in the
    background while the GPU proves (the TallRefs pattern of test_gpu_height_range)"""

    def __init__(self, orc):
        self.segments = {k: _segment_chip(orc, k) for k in SEGMENTS}
        self.mix = _chips(TALL_MIX, seed=61)
        self.fast = orc.fast_available()
        self._pool = self._futures = None
        if self.fast:
            self._pool = ThreadPoolExecutor(2)
            self._futures = {k: self._pool.submit(lambda c: orc.prove(*c, fast=True)[:3], c) for k, c in self.segments.items()}
            self._futures["mix"] = self._pool.submit(lambda: orc.prove_chips(self.mix, fast=True))

    def ref(self, key):
        return self._futures[key].result() if self.fast else None

    def close(self):
        if self._pool is not None:
            self._pool.shutdown(cancel_futures=True)


@pytest.fixture(scope="module")
def scale(orc):
    r = ScaleRefs(orc)
    yield r
    r.close()


def test_every_segment_reaches_every_block_count(orc):
    """the budgets of 2. pick 2, 4, 8 and 16 blocks in turn: blocking saves more than the blocked quotient costs"""
    for name, (_, on_device) in SEGMENTS.items():
        shp = shapes(orc, [_segment_chip(orc, name)])
        for lb in range(1, 5):
            budget_for(shp, lb, shp[0][0] + 1, not on_device)
    assert orc.Air(*_segment_chip(orc, "2p14_perm_140")[1:]).perm_width == 140


@gpu
@pytest.mark.parametrize("name", list(SEGMENTS))
def test_blocked_segment_at_scale_equals_the_resident_segment(ctx, orc, scale, name):
    """proof, cumulative sum, opened values and query words in 2, 4, 8 and 16 blocks = the resident proof of the same context, which
    equals the oracle's"""
    trace, bc, spans, bus = chip = scale.segments[name]
    on_device = SEGMENTS[name][1]
    w, n = trace.shape
    log_n = n.bit_length() - 1
    shp = shapes(orc, [chip])
    air = ctx.air(bc, spans, w, bus)
    d = host = None
    try:
        if on_device:
            d = ctx.to_device(trace)
            src = d.ptr
        else:                                     # pinned Montgomery words
            m = _mont(trace)
            host = ctx.host_alloc(m.nbytes)
            C.memmove(host, m.ctypes.data, m.nbytes)
            src = host

        def prove(budget):
            ctx.set_memory_budget(budget)
            try:
                proof = ctx.prove_segment(air, src, log_n, w, on_device=on_device)
                lb = ctx.last_row_blocks()
            finally:
                ctx.set_memory_budget(0)
            q, ys = ctx.query_segment(log_n, w, air.perm_width)
            return proof, ys, q, lb

        ref = prove(0)
        assert ref[3] == 0
        for lb in range(1, 5):
            got = prove(budget_for(shp, lb, log_n + 1, not on_device))
            assert got[3] == lb
            assert got[0] == ref[0], lb
            assert (got[1] == ref[1]).all() and (got[2] == ref[2]).all(), lb
    finally:
        air.free()
        if d is not None:
            d.free()
        if host:
            ctx.host_free(host)
    proof, ys, q, _ = ref
    if scale.fast:
        e_proof, e_ys, e_q = scale.ref(name)
        assert proof == e_proof and (ys == e_ys).all() and (q == e_q).all()
    else:
        assert orc.verify_segment(bc, spans, log_n, w, proof, ys, q, bus=bus) == 0
        _sampled_checks(ctx, orc, chip, n_lde_checks=1)


# ---------------------------------------------------------------- 3. a tall mix at every pair choose_row_blocks can pick
def _mix_choices(shp):
    """every (lb, lowest blocked height) some budget makes choose_row_blocks pick, each with such a budget"""
    heights = sorted({s[0] + 1 for s in shp}, reverse=True)
    out = {}
    for lb in range(1, 5):
        for h in heights:
            if h < lb + 4:
                break
            b = footprint(shp, lb, h)
            c = choice(shp, b)
            if c not in out:
                out[c] = b
    return out


def test_the_tall_mix_reaches_every_block_count_and_cut(orc):
    shp = shapes(orc, _chips(TALL_MIX, seed=61))
    assert shp[2][2] == 0 and shp[1][2] > 0                      # two chips at 2^18, one without interactions
    got = _mix_choices(shp)
    assert {lb for lb, _ in got} == {1, 2, 3, 4}
    assert len(got) >= 10, sorted(got)
    assert (4, 8) in got                                         # 16 blocks down to the 2^7 chip


@gpu
def test_tall_mix_at_every_choice_equals_the_resident_proof(ctx, orc, scale):
    """heights 2^20, 2^18 (two chips, one without interactions), 2^14, 2^7 and 2^2 (never blocked)"""
    shp = shapes(orc, scale.mix)
    cs = ChipSet(ctx, scale.mix)
    try:
        ref, lb0 = cs.prove(0)
        assert lb0 == 0
        for (lb, h), budget in sorted(_mix_choices(shp).items()):
            got, lb_got = cs.prove(budget)
            assert lb_got == lb, (lb, h)
            _assert_same(got, ref, (lb, h))
    finally:
        cs.free()
    if scale.fast:
        _assert_same(ref, scale.ref("mix"), "oracle")
    else:
        assert orc.verify_chips(scale.mix, *ref, check_constraints=False) == 0


# ---------------------------------------------------------------- 4. query phases that skip blocks
SKIP_SPEC = [(16, 10, 2, 6), (14, 8, 1, 4)]
SKIP_SEED = 94              # its queries fall into blocks 0, 11, 11 (asserted)


def _blocks_hit(q, log_max, lb):
    """the block of each query index: row r >> (log_max - log_h) of height 2^log_h lies in block that >> (log_h - lb), for every
    blocked height the same block"""
    return [int(r) >> (log_max - lb) for r in q[:, 0]]


@gpu
def test_query_phases_that_skip_blocks_equal_the_resident_ones(ctx, orc):
    """16 blocks of a 2^16 chip and of a blocked 2^14 chip under it, 1, 2 and 3 queries: separate proofs in one context, so that a
    block left in a chip's buffer by the reduced opening or by an earlier query phase would show.  The resident proofs run in a
    context of their own: a query word the blocked phase fails to write must not find the right value left in the output buffer."""
    import powdr_b200
    chips = _chips(SKIP_SPEC, seed=SKIP_SEED)
    shp = shapes(orc, chips)
    budget = budget_for(shp, 4, 15)
    refs = {}
    c2 = powdr_b200.Context(0)
    try:
        res = ChipSet(c2, chips)
        try:
            for nq in (1, 2, 3):
                c2.set_fri_params(nq, 4)
                refs[nq], _ = res.prove(0)
        finally:
            res.free()
    finally:
        c2.close()
    cs = ChipSet(ctx, chips)
    hits = []
    try:
        for nq in (1, 2, 3, 1):
            ctx.set_fri_params(nq, 4)
            got, lb = cs.prove(budget)
            assert lb == 4
            _assert_same(got, refs[nq], nq)
            hits.append(_blocks_hit(got[3], 17, 4))
    finally:
        ctx.set_fri_params(8, 4)
        cs.free()
    assert all(len(set(h)) < 16 for h in hits)
    assert len(hits[2]) == 3 and len(set(hits[2])) == 2, ("not two queries in one block", hits[2])
    e = orc.prove_chips(chips, n_queries=3, pow_bits=4)
    _assert_same(refs[3], e, "oracle")


# ---------------------------------------------------------------- 5. twiddle-cache churn
CHURN_SPEC = [(12, 6, 1, 3), (11, 5, 0, 2), (10, 7, 2, 2), (9, 4, 1, 2), (8, 6, 0, 3), (7, 5, 1, 2)]


def test_the_churn_mix_blocks_six_heights_in_16_blocks(orc):
    shp = shapes(orc, _chips(CHURN_SPEC, seed=80))
    budget_for(shp, 4, 8)
    assert 16 * len(shp) > 64                     # block twiddle sets (one per block shift and height) beyond the FIFO's 64


@gpu
def test_twiddle_cache_churn_in_one_proof(orc):
    """six blocked heights at 16 blocks create 96 block twiddle sets in one proof, so get_twiddles evicts sets the proof still uses;
    a second proof starts from that warm, partly evicted cache"""
    import powdr_b200
    chips = _chips(CHURN_SPEC, seed=80)
    shp = shapes(orc, chips)
    c2 = powdr_b200.Context(0)
    try:
        c2.set_fri_params(8, 4)
        cs = ChipSet(c2, chips)
        try:
            ref, _ = cs.prove(0)
            for i in range(2):
                got, lb = cs.prove(budget_for(shp, 4, 8))
                assert lb == 4
                _assert_same(got, ref, "proof %d" % i)
        finally:
            cs.free()
    finally:
        c2.close()
    _assert_same(ref, orc.prove_chips(chips, n_queries=8, pow_bits=4), "oracle")


# ---------------------------------------------------------------- 6. blocked against sharded
@gpu
@pytest.mark.parametrize("world", [4, 16])
def test_blocked_segment_equals_the_sharded_segment(ctx, orc, world):
    """B row blocks on one GPU = B thread-ranks of pb_prove_segment_sharded (ThreadComm, one GPU): the same sub-coset blocks, folded
    for every destination block at once on the ranks, one at a time here"""
    from powdr_b200.sharded import prove_segment_threads
    lb, log_n = world.bit_length() - 1, 10
    chip = _chips([(log_n, 9, 2, 5)], seed=90 + world)[0]
    trace, bc, spans, bus = chip
    air = ctx.air(bc, spans, trace.shape[0], bus)
    d = ctx.to_device(trace)
    try:
        ctx.set_memory_budget(budget_for(shapes(orc, [chip]), lb, log_n + 1))
        proof = ctx.prove_segment(air, d.ptr, log_n, trace.shape[0], on_device=True)
        assert ctx.last_row_blocks() == lb
        q, _ = ctx.query_segment(log_n, trace.shape[0], air.perm_width)
    finally:
        ctx.set_memory_budget(0)
        air.free()
        d.free()
    ranks = prove_segment_threads(world, trace, bc, spans, bus=bus, want_queries=True)
    for r, (p, rq) in enumerate(ranks):
        assert p == proof and (rq == q).all(), r


KECCAK_LOG_N, KECCAK_WIDTH, KECCAK_INTS, KECCAK_WORLD = 21, 2022, 1734, 4


@gpu
def test_keccak_shape_at_2p21_rows_blocked_equals_sharded(orc):
    """2^21 x 2022 with 1734 interactions (test_keccak_logup_shape_at_2p21_rows_beyond_hbm) in 8 and 16 row blocks on one GPU, then
    pb_prove_segment_sharded on 4 GPUs, whose proof is the single-GPU proof: proof, opened values and query words word for word"""
    import torch
    import powdr_b200
    from powdr_b200 import machine as M
    from powdr_b200.sharded import ThreadComm, _run_ranks, shard_columns
    n_dev = torch.cuda.device_count()
    if n_dev < KECCAK_WORLD:
        pytest.skip("the sharded proof of the 2^21 x 2022 segment takes %d GPUs (a quarter of its 113 GiB of matrices each); %d visible"
                    % (KECCAK_WORLD, n_dev))
    log_n = KECCAK_LOG_N
    mach = M.SymbolicMachine([], M.synthetic_bus(KECCAK_WIDTH, KECCAK_INTS, seed=0xB2000002))
    w = mach.width
    bus = M.compile_bus(mach, 1)
    gen = torch.Generator(device="cuda:0").manual_seed(0xB2000021)
    trace = torch.randint(0, P, (w, 1 << log_n), dtype=torch.int32, device="cuda:0", generator=gen)
    single = powdr_b200.Context(0)                    # its workspaces are freed before the ranks start
    try:
        single.set_fri_params(8, 4)
        air = single.air([], [], w, bus)
        wp = air.perm_width
        assert single.lib.pb_to_monty(single.h, C.c_void_p(trace.data_ptr()), C.c_size_t(trace.numel())) == 0
        single.synchronize()
        blocked = []
        for lb in (3, 4):
            single.set_memory_budget(footprint([(log_n, w, wp)], lb))
            proof = single.prove_segment(air, trace.data_ptr(), log_n, w, on_device=True)
            assert single.last_row_blocks() == lb
            q, ys = single.query_segment(log_n, w, wp)
            blocked.append((proof, ys, q))
        single.set_memory_budget(0)
        assert blocked[0][0] == blocked[1][0] and (blocked[0][1] == blocked[1][1]).all() and (blocked[0][2] == blocked[1][2]).all()
        air.free()
        # each rank's column block on its own device (Montgomery words, as the sharded prover takes them)
        cols = []
        for r in range(KECCAK_WORLD):
            f, k = shard_columns(w, KECCAK_WORLD, r)
            cols.append(trace[f:f + k].to("cuda:%d" % r, copy=True) if k else None)
    finally:
        single.close()
        del trace
        torch.cuda.empty_cache()
    proof, ys, q = blocked[0]

    def body(rank, group):
        c = powdr_b200.Context(rank)
        try:
            c.set_fri_params(8, 4)
            a = c.air([], [], w, bus)
            comm = ThreadComm(group, rank, c)
            blk = cols[rank]
            p = c.prove_segment_sharded(a, blk.data_ptr() if blk is not None else 0, log_n, w, comm, on_device=True)
            rq = c.query_segment_sharded(comm, log_n, w, a.perm_width)
            rys = np.empty(ys.shape, dtype=np.uint32)
            assert c.lib.pb_last_openings(c.h, rys.ctypes.data_as(C.c_void_p), C.c_size_t(rys.size)) == 0
            if comm.error:
                raise comm.error
            a.free()
            return p, rys, rq
        finally:
            c.close()

    try:
        ranks = _run_ranks(KECCAK_WORLD, body)
    finally:
        del cols
        torch.cuda.empty_cache()
    for r, (p, rys, rq) in enumerate(ranks):
        assert p == proof, r
        assert (rys == ys).all(), r
        assert (rq == q).all(), r
