"""CPU checks of the footprint the single-GPU provers choose their path by (pb_footprint_bytes, include/powdr_b200.h) and of the kernel
the row-blocked openings add."""
from powdr_b200.capi import footprint_bytes

from test_kernel_resources import resource_usage

KECCAK = (2022, 3348)          # the headline APC chip: 2022 columns, 1734 interactions -> 3348 permutation columns


def test_the_matrices_of_the_keccak_shape_follow_the_accounting():
    w, wp = KECCAK
    for log_n in (20, 21):
        n = 1 << log_n
        fp = [footprint_bytes([(log_n, w, wp)], lb) for lb in range(5)]
        # resident: main LDE (2N x W), permutation trace and its LDE (3N x W_p); blocked: coefficients + one of B blocks of each LDE
        big = [4 * (2 * n * w + 3 * n * wp)] + [4 * (n * (w + wp) + (2 * n >> lb) * (w + wp)) for lb in range(1, 5)]
        small = [f - b for f, b in zip(fp, big)]
        assert all(0 < s < 4 << 30 for s in small), small          # trees, quotient, FRI, scratch: below 4 GiB
        assert fp == sorted(fp, reverse=True)
    assert footprint_bytes([(20, w, wp)], 0) < 79 << 30              # an idle 80 GB card keeps the resident path
    assert 55e9 < footprint_bytes([(21, w, wp)], 3) < 61e9            # 2^21 rows in 8 blocks: ~58 GB beside the 17 GB trace
    assert footprint_bytes([(21, w, wp)], 0) > 110 << 30


def test_heights_too_short_for_the_blocks_stay_whole():
    # log_n >= log_blocks + 3: at 16 blocks a 2^6 chip keeps its resident LDE, at 2 blocks it is blocked
    tall, short = (12, 64, 40), (6, 64, 40)
    d16 = footprint_bytes([tall, short], 4) - footprint_bytes([tall], 4)
    assert d16 - 4 * (2 * 64 * 64 + 3 * 64 * 40) in range(0, 4 * 64 * 64)
    assert footprint_bytes([short], 1) < footprint_bytes([short], 0)


def test_monomial_weights_kernel_has_no_stack_frame_or_local_memory():
    usage = {n: u for n, u in resource_usage().items() if "monomial_weights_kernel" in n}
    assert len(usage) == 1 and all(u[1] == 0 and u[2] == 0 for u in usage.values()), usage
