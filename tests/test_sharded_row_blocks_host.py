"""CPU checks of the footprint the sharded provers choose their path by (pb_footprint_bytes_sharded, include/powdr_b200.h): a Python
restatement of the accounting equals the library, and the restated choice reaches every (world, sub-blocks, lowest blocked height)."""
import pytest

from powdr_b200.capi import footprint_bytes_sharded

SMS, RESERVE = 132, 64 << 20
KECCAK = (2022, 3348)          # the headline APC chip: 2022 columns, 1734 interactions -> 3348 permutation columns


def footprint_sharded(chips, world, lb, h_cut=0, host_trace=False):
    """one rank's bytes: chips [(log_n, width, perm_width)], heights log_n + 1 >= h_cut with log_n >= g + lb + 3 in 2^lb sub-blocks"""
    G, g = world, world.bit_length() - 1
    words = n_max = hmax = hperm = scratch = sub = 0
    s_main = s_plde = s_rows = s_perm = s_sp = s_q = s_qw = 0
    xb = {}
    any_bl = False
    for log_n, w, wp in chips:
        n = 1 << log_n
        ms, rows_t, per, perp = 2 * n // G, n // G, -(-w // G), -(-wp // G)
        bl = lb > 0 and log_n + 1 >= h_cut and log_n >= g + lb + 3
        mb = ms >> (lb if bl else 0)
        words += w * mb + (per * n if bl else 0)                 # main LDE sub-block, coefficients of my columns
        words += 8 * n + 8 * ms                                   # quotient chunks, my block of their LDE
        if wp:
            words += 2 * perp * n + 4 * rows_t + wp * mb          # rows x perm columns | row sums | my perm columns; perm LDE
        if bl:
            any_bl = True
            xb[(log_n, 0)] = xb.get((log_n, 0), 0) + per * mb
            xb[(log_n, 1)] = xb.get((log_n, 1), 0) + perp * mb
            sub = max(sub, 12 * mb)
        else:
            s_main += per * ms
            s_plde += perp * ms
        if wp:
            s_rows += per * rows_t
            s_perm += perp * rows_t
            s_sp += 8 * ms
            hperm = max(hperm, log_n + 1)
        s_q += 4 * ms
        s_qw += 8 * n
        n_max, hmax = max(n_max, n), max(hmax, log_n + 1)
        scratch = max(scratch, 3 * min(max(per, perp, 8) * n, max(n, (16 * SMS) << 15)))
    x = max([s_main, s_plde, s_rows, s_perm, s_q] + list(xb.values()))
    words += 2 * G * x
    m = 1 << (hmax - g)
    words += 32 * m + (16 << (hperm - g) if hperm else 0) + 8 * m
    words += s_sp // 2 + s_sp * (1 + G) + s_qw
    if any_bl:
        words += s_q + sub
    words += 4 * (2 * n_max // G) + scratch + 4 * (2 * n_max // G) + 4 * n_max
    words += 28 * m + 8 * n_max + 32 * n_max
    if host_trace:
        words += -(-chips[0][1] // G) * n_max
    return 4 * words + RESERVE


def choose(chips, world, budget):
    """the sharded provers' path: None resident, (lb, lowest blocked LDE height), or "none" when nothing fits"""
    if not budget or footprint_sharded(chips, world, 0) <= budget:
        return None
    g = world.bit_length() - 1
    heights = sorted({c[0] + 1 for c in chips}, reverse=True)
    lb = 1
    while world << lb <= 16:
        for h in heights:
            if h < g + lb + 4:
                break
            if footprint_sharded(chips, world, lb, h) <= budget:
                return lb, h
        lb += 1
    return "none"


# LDE heights 2^15, 2^11, 2^9, 2^7 (the last too short for any blocking at 16 blocks): the tallest dominates, and every height has a
# permutation trace wider than its main trace, so that blocking a height saves memory even at 2 sub-blocks (which free as much of the
# main LDE block as the kept coefficients of my columns take)
MIX = [(14, 16, 48), (10, 12, 40), (8, 10, 32), (6, 9, 8)]


def _allowed(world):
    return [lb for lb in range(4) if world << lb <= 16]


@pytest.mark.parametrize("world", [2, 4, 8])
def test_restated_footprint_equals_the_library(world):
    shapes = [MIX, [(21,) + KECCAK], [(20,) + KECCAK], [(7, 5, 0)], [(9, 3, 8), (9, 12, 0), (7, 2, 0)]]
    for chips in shapes:
        for lb in _allowed(world):
            assert footprint_bytes_sharded(chips, world, lb) == footprint_sharded(chips, world, lb), (chips, world, lb)


def test_the_library_refuses_what_the_sharded_provers_do_not_run():
    from powdr_b200.capi import PbError
    for world, lb, chips in ((3, 0, MIX), (16, 1, MIX), (2, 4, MIX), (4, 3, MIX), (8, 0, [(5, 4, 0)])):
        with pytest.raises(PbError):
            footprint_bytes_sharded(chips, world, lb)


@pytest.mark.parametrize("world", [2, 4, 8])
def test_the_restated_choice_reaches_every_blocking(world):
    g = world.bit_length() - 1
    seen = set()
    assert choose(MIX, world, 0) is None
    assert choose(MIX, world, footprint_sharded(MIX, world, 0)) is None
    for lb in _allowed(world)[1:]:
        for h in sorted({c[0] + 1 for c in MIX}, reverse=True):
            if h < g + lb + 4:
                continue
            got = choose(MIX, world, footprint_sharded(MIX, world, lb, h))
            assert got == (lb, h), (world, lb, h, got)
            seen.add(got)
    # every (sub-blocks, lowest blocked height) pair the rule allows: log_n >= g + lb + 3
    assert seen == {(lb, c[0] + 1) for lb in _allowed(world)[1:] for c in MIX if c[0] >= g + lb + 3}
    smallest = min(footprint_sharded(MIX, world, lb, 0) for lb in _allowed(world))
    assert choose(MIX, world, smallest - 1) == "none"


def test_the_keccak_shapes_per_rank():
    w, wp = KECCAK
    gb = 1e9
    # 2^20 rows on 2 ranks: every sub-block count shrinks the footprint, and each fits an 80 GB card beside the 4.2 GB column share
    assert 40 * gb < footprint_sharded([(20, w, wp)], 2, 0) < 75 * gb
    assert footprint_sharded([(20, w, wp)], 2, 2) < footprint_sharded([(20, w, wp)], 2, 1) < footprint_sharded([(20, w, wp)], 2, 0)
    # 2^21 rows on 2 ranks, an 80 GB-class card (79 GiB usable, as for one GPU) less the 8.5 GB column share: B = 8 fits, B = 4 does not
    share = 4 * 1011 * (1 << 21)
    budget = (79 << 30) - share
    assert choose([(21, w, wp)], 2, budget) == (3, 22)
    assert footprint_sharded([(21, w, wp)], 2, 3) + share < 79 << 30 < footprint_sharded([(21, w, wp)], 2, 2) + share
    assert footprint_bytes_sharded([(21, w, wp)], 2, 3) == footprint_sharded([(21, w, wp)], 2, 3)
    # blocking shrinks the LDE sub-blocks; the LogUp-phase rows, permutation columns and their exchange buffers stay
    for world in (2, 4):
        fp = [footprint_sharded([(21, w, wp)], world, lb) for lb in _allowed(world)]
        assert fp == sorted(fp, reverse=True), fp
