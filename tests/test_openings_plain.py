"""The oracle's openings, DEEP reduced opening and FRI fold against the plain reference (tests/py_openings.py), both the
scalar restatement and the AVX-512 arm, at the points where a formula over the domain goes wrong: zeta on the trace domain,
zeta 0, 1 and with a single non-zero limb, gamma and beta 0, 1 and p-1, and the edge columns the GPU kernels carry.
At 16 rows and more, so that the AVX-512 arm does not fall back to the scalar one."""
import numpy as np
import pytest

import py_openings as ref
from util import P, rand_field


@pytest.fixture(scope="module")
def fast(orc):
    if not orc.fast_available():
        pytest.skip("host CPU has no AVX-512")
    return orc


# ---------------------------------------------------------------- the reference against itself
def test_reference_field_and_domain():
    rng = np.random.default_rng(1)
    for _ in range(20):
        a = tuple(int(x) for x in rng.integers(0, P, 4))
        assert ref.e4_mul(a, ref.e4_inv(a)) == ref.ONE
        assert ref.e4_mul(a, ref.e4_pow(a, 5)) == ref.e4_pow(a, 6)
    x4 = ref.e4_pow((0, 1, 0, 0), 4)
    assert x4 == (11, 0, 0, 0)
    for log_n in (1, 5, 27):
        w = ref.root_of_unity(log_n)
        assert pow(w, 1 << log_n, P) == 1 and pow(w, 1 << (log_n - 1), P) == P - 1
    for log_n, br in ((5, False), (5, True), (0, True), (9, True)):
        g = ref.geom(7, log_n, br)
        assert g.tolist() == [pow(7, ref.bitrev(i, log_n) if br else i, P) for i in range(1 << log_n)]
    a = rand_field(rng, (4, 33)).astype(np.uint64)
    inv = ref.e4_inv_np(a)
    for i in range(33):
        assert tuple(int(x) for x in inv[:, i]) == ref.e4_inv(tuple(int(x) for x in a[:, i]))
    assert ref.in_coset((31 * pow(ref.root_of_unity(6), 5, P) % P, 0, 0, 0), 31, 6)
    assert not ref.in_coset((31, 1, 0, 0), 31, 6) and not ref.in_coset(ref.ONE, 31, 6) and ref.in_coset(ref.ONE, P - 1, 6)


def test_reference_openings_agree():
    """closed form of a sparse polynomial = interpolation + Horner = Lagrange closed form, at every kind of point"""
    rng = np.random.default_rng(2)
    log_n = 6
    n = 1 << log_n
    terms = [(0, 5), (1, P - 1), (n - 1, 123456789), (17, 3)]
    for shift in ref.SHIFTS:
        col = ref.sparse_codeword(terms, log_n, shift)
        assert not col[1:].any()
        col = col[0]
        spike = np.zeros(n, dtype=np.uint64)
        spike[9] = P - 1
        for name, z, row in ref.zeta_cases(log_n, shift, rng):
            exp = ref.eval_sparse(terms, z)
            assert ref.eval_dense(col, shift, z) == exp, name
            if row is not None:
                assert exp == (int(col[row]), 0, 0, 0), name
            lag = ref.e4_scale(ref.lagrange_at(log_n, shift, 9, z), P - 1)
            assert ref.eval_dense(spike, shift, z) == lag, name


def test_reference_fold_and_deep_agree():
    rng = np.random.default_rng(3)
    log_len = 5
    terms = [(0, (1, 2, 3, 4)), (1, (P - 1, 0, 0, 7)), (6, 9), (31, (5, 6, 7, 8))]
    beta = (11, 22, 33, 44)
    shift = 31
    cw = ref.sparse_codeword(terms, log_len, shift, bit_reversed=True)
    xs = ref.geom(ref.root_of_unity(log_len), log_len - 1, bit_reversed=True) * shift % P       # x_j = shift w_len^bitrev(j)
    folded = ref.sparse_codeword(ref.fold_sparse(terms, beta), log_len - 1, shift * shift % P, bit_reversed=True)
    for j in range(1 << (log_len - 1)):
        lo, hi = tuple(int(v) for v in cw[:, 2 * j]), tuple(int(v) for v in cw[:, 2 * j + 1])
        assert ref.fold_pair(lo, hi, int(xs[j]), beta) == tuple(int(v) for v in folded[:, j])
    cols = rand_field(rng, (5, 16))
    ys = [tuple(int(v) for v in y) for y in rand_field(rng, (5, 4))]
    gamma, zeta = (3, 1, 4, 1), (5, 9, 2, 6)
    xs = ref.domain_np(4, 31, bit_reversed=True)
    gp = ref.gamma_powers(gamma, 5)
    ysum = ref.ZERO
    for g, y in zip(gp, ys):
        ysum = ref.e4_add(ysum, ref.e4_mul(g, y))
    got = ref.deep_rows_np(cols, gp, ysum, xs, zeta)
    for r in range(16):
        assert tuple(int(v) for v in got[:, r]) == ref.deep_row(cols[:, r].tolist(), ys, gamma, int(xs[r]), zeta)


# ---------------------------------------------------------------- openings
@pytest.mark.parametrize("log_n", [4, 5, 6, 9])
def test_eval_at_point_edges(orc, log_n):
    rng = np.random.default_rng(10 + log_n)
    mat, expected = ref.edge_columns(log_n, rng)
    impls = [("orc", orc.eval_at_point)] + ([("fast", orc.fast_eval_at_point)] if orc.fast_available() else [])
    for shift in ref.SHIFTS:
        for name, z, row in ref.zeta_cases(log_n, shift, rng):
            exp = expected(shift, z)
            if row is not None:
                assert exp == [(int(v), 0, 0, 0) for v in mat[:, row]]
            for impl, f in impls:
                got = [tuple(int(v) for v in y) for y in f(mat, shift, z)]
                assert got == exp, (impl, shift, name)


@pytest.mark.parametrize("log_n", [4, 7])
def test_eval_at_point_dense(orc, log_n):
    rng = np.random.default_rng(20 + log_n)
    mat = rand_field(rng, (3, 1 << log_n))
    mat[1, ::3] = P - 1
    for shift in (31, 1234567):
        coefs = [ref.interpolate(c) for c in mat]
        for name, z, row in ref.zeta_cases(log_n, shift, rng):
            zs = ref.e4_scale(z, pow(shift, P - 2, P))
            exp = [ref.horner(c, zs) for c in coefs]
            assert [tuple(int(v) for v in y) for y in orc.eval_at_point(mat, shift, z)] == exp, name
            if orc.fast_available():
                assert [tuple(int(v) for v in y) for y in orc.fast_eval_at_point(mat, shift, z)] == exp, name


def test_fast_eval_at_point_in_domain_large(fast):
    """the AVX-512 arm at 2^12 rows, at the points of the domain, where its batch inversion meets a zero denominator"""
    log_n = 12
    rng = np.random.default_rng(4)
    mat = rand_field(rng, (2, 1 << log_n))
    for i in (0, 1, 63, 64, 2047, 4095):
        z = (ref.domain_point(31, log_n, i), 0, 0, 0)
        assert (fast.fast_eval_at_point(mat, 31, z) == np.array([[mat[0, i], 0, 0, 0], [mat[1, i], 0, 0, 0]])).all()


# ---------------------------------------------------------------- DEEP reduced opening
GAMMAS = {"0": ref.ZERO, "1": ref.ONE, "p-1": (P - 1, 0, 0, 0), "base": (987654321, 0, 0, 0), "ext4": (1234, 5678, 91011, 121314)}


def _deep_expected(mats, shift, zeta, gamma, ys):
    cols = np.concatenate(mats, axis=0)
    m = cols.shape[1]
    gp = ref.gamma_powers(gamma, cols.shape[0])
    ysum = ref.ZERO
    for g, y in zip(gp, ys):
        ysum = ref.e4_add(ysum, ref.e4_mul(g, ref.e4(y)))
    xs = ref.domain_np(m.bit_length() - 1, shift, bit_reversed=True)
    return ref.deep_rows_np(cols, gp, ysum, xs, zeta).T.astype(np.uint32)


@pytest.mark.parametrize("log_m,widths", [(4, [1]), (5, [3, 5]), (7, [8, 1, 9]), (10, [17])])
def test_deep_quotient(orc, log_m, widths):
    rng = np.random.default_rng(30 + log_m)
    m = 1 << log_m
    mats = [rand_field(rng, (w, m)) for w in widths]
    mats[0][0, :] = P - 1
    ys = rand_field(rng, (sum(widths), 4))
    impls = [("orc", orc.deep_quotient)] + ([("fast", orc.fast_deep_quotient)] if orc.fast_available() else [])
    zetas = [(1, 2, 3, 4), (5, 0, 0, 0), (0, 0, 0, 9), ref.ZERO, ((P - 1), (P - 1), (P - 1), (P - 1)),
             (ref.domain_point(1, log_m, 3), 0, 0, 0)]            # a point of H: the LDE coset is 31*H', disjoint from it
    for shift in (31, 1234567):
        for gname, gamma in GAMMAS.items():
            for zeta in zetas:
                assert not ref.in_coset(zeta, shift, log_m)
                exp = _deep_expected(mats, shift, zeta, gamma, ys)
                for impl, f in impls:
                    assert (f(mats, shift, zeta, gamma, ys) == exp).all(), (impl, shift, gname, zeta)


@pytest.mark.parametrize("log_m", [4, 7])
def test_deep_quotient_refuses_points_of_the_lde_domain(orc, log_m):
    """(x_r - zeta)^-1 does not exist at the row where x_r = zeta: both arms refuse rather than return a value"""
    rng = np.random.default_rng(40 + log_m)
    m = 1 << log_m
    mats = [rand_field(rng, (3, m))]
    ys = rand_field(rng, (3, 4))
    impls = [orc.deep_quotient] + ([orc.fast_deep_quotient] if orc.fast_available() else [])
    for shift in (31, P - 1):
        for r in (0, 9, m - 1):
            zeta = (ref.domain_point(shift, log_m, r), 0, 0, 0)
            for f in impls:
                with pytest.raises(ValueError):
                    f(mats, shift, zeta, (3, 0, 0, 0), ys)


# ---------------------------------------------------------------- FRI fold
BETAS = {"0": ref.ZERO, "1": ref.ONE, "p-1": (P - 1, 0, 0, 0), "base": (555555555, 0, 0, 0), "ext4": (P - 2, 3, P - 4, 5)}


@pytest.mark.parametrize("log_len", list(range(1, 13)))
def test_fri_fold(orc, log_len):
    rng = np.random.default_rng(50 + log_len)
    n = 1 << log_len
    terms = [(0, (1, 2, 3, 4)), (1, (P - 1,) * 4), (n - 1, tuple(int(x) for x in rng.integers(0, P, 4))), (int(rng.integers(0, n)), 7)]
    for shift in (1, 31, P - 1, pow(31, 1 << (log_len % 5), P)):
        cw = ref.sparse_codeword(terms, log_len, shift, bit_reversed=True).T.astype(np.uint32)
        for bname, beta in BETAS.items():
            exp = ref.sparse_codeword(ref.fold_sparse(terms, beta), log_len - 1, shift * shift % P, bit_reversed=True).T
            assert (orc.fri_fold(cw, shift, beta) == exp).all(), (shift, bname)
    full = np.full((n, 4), P - 1, dtype=np.uint32)
    assert (orc.fri_fold(full, 31, BETAS["ext4"]) == P - 1).all()
