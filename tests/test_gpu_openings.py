"""pb_eval_at_point, pb_deep_quotient and pb_fri_fold against the plain reference (tests/py_openings.py), word for word on the
raw device words, at every launch geometry of their kernels and at the points where a formula over the domain goes wrong.

- openings: heights that give 1, 2, 4 and 512 row splits of eval_partial_kernel, every width % EV_COLS, sparse-polynomial
  columns (closed form at any height), all p-1 columns (the 96-bit accumulators at their largest), p-1 spikes at the CTA and
  split boundaries, and zeta on the trace domain itself;
- reduced opening: partial last CTAs, 1 to 513 columns per run against the 8-column pipeline and the 256-column gamma chunks,
  1 to 17 runs (one launch per 8 runs, the later ones accumulate), runs that must be merged, and zeta on the LDE domain refused;
- fold: every length from 2 to 2^25, the twiddle-table cache, and fold chains that end in the closed-form constant."""
import numpy as np
import pytest

import py_openings as ref
from util import P, rand_field

pytestmark = pytest.mark.gpu

R_MOD_P = (1 << 32) % P
_P64 = np.uint64(P)


def _monty(a):
    return (np.asarray(a, dtype=np.uint64) * np.uint64(R_MOD_P) % _P64).astype(np.uint32)


def _raw_upload(ctx, a):
    a = np.ascontiguousarray(a, dtype=np.uint32)
    return ctx.alloc(a.nbytes).upload(a)


def _guarded_out(ctx, n_words, guard=16):
    """device output with `guard` words of 0xFFFFFFFF behind it (the kernels must not write there)"""
    return _raw_upload(ctx, np.full(n_words + guard, 0xFFFFFFFF, dtype=np.uint32))


# ---------------------------------------------------------------- pb_eval_at_point
EVAL_LOGS = [1, 2, 7, 8, 9, 10, 15, 16, 17, 20, 24]
WIDTHS = [1, 2, 3, 4, 5, 7, 9]


def _eval(ctx, d_mat, log_n, width, shift, zeta):
    d_ys = _guarded_out(ctx, 4 * width)
    ctx.eval_at_point(d_mat.ptr, log_n, width, shift, zeta, d_ys.ptr)
    raw = d_ys.download(4 * width + 16)
    assert (raw[4 * width:] == 0xFFFFFFFF).all(), "pb_eval_at_point wrote past d_ys[width]"
    return raw[:4 * width].reshape(width, 4)


@pytest.mark.parametrize("log_n", EVAL_LOGS)
def test_eval_at_point_edges(ctx, log_n):
    rng = np.random.default_rng(100 + log_n)
    mat, expected = ref.edge_columns(log_n, rng)
    width = mat.shape[0]
    d_mat = ctx.to_device(mat)
    n_cases = 0
    for shift in ref.SHIFTS:
        for name, z, row in ref.zeta_cases(log_n, shift, rng):
            exp = expected(shift, z)
            if row is not None:
                assert exp == [(int(v), 0, 0, 0) for v in mat[:, row]]
            got = _eval(ctx, d_mat, log_n, width, shift, z)
            assert (got == _monty(exp)).all(), (shift, name, [k for k in range(width) if not (got[k] == _monty(exp[k])).all()])
            n_cases += 1
    # every width % EV_COLS, on the leading columns of the same matrix
    for w in WIDTHS:
        if w > width:
            continue
        for z in [tuple(int(x) for x in rng.integers(0, P, 4)), (ref.domain_point(31, log_n, (1 << log_n) - 1), 0, 0, 0)]:
            got = _eval(ctx, d_mat, log_n, w, 31, z)
            assert (got == _monty(expected(31, z)[:w])).all(), (w, z)
    assert n_cases >= 40


@pytest.mark.parametrize("log_n", [1, 4, 8, 10])
def test_eval_at_point_dense(ctx, log_n):
    """random columns against interpolation + Horner"""
    rng = np.random.default_rng(200 + log_n)
    mat = rand_field(rng, (5, 1 << log_n))
    mat[0, :] = P - 1
    mat[1, ::2] = 0
    coefs = [ref.interpolate(c) for c in mat]
    d_mat = ctx.to_device(mat)
    for shift in ref.SHIFTS:
        inv_shift = pow(shift, P - 2, P)
        for name, z, row in ref.zeta_cases(log_n, shift, rng):
            exp = [ref.horner(c, ref.e4_scale(z, inv_shift)) for c in coefs]
            assert (_eval(ctx, d_mat, log_n, 5, shift, z) == _monty(exp)).all(), (shift, name)


# ---------------------------------------------------------------- pb_deep_quotient
DQ_LOGS = [1, 2, 7, 8, 9, 13, 16, 20]
COUNTS = [1, 7, 8, 15, 16, 17, 255, 256, 257, 513]
GAMMAS = [("0", ref.ZERO), ("1", ref.ONE), ("p-1", (P - 1, 0, 0, 0)), ("base", (987654321, 0, 0, 0)), ("ext4", (1234, 5678, 91011, 121314))]


def _layouts(log_m):
    """(name, columns per run): each run a separate matrix, unless merged"""
    if log_m <= 13:
        out = [("run%d" % c, [c]) for c in COUNTS]
        out += [("8runs", [1, 7, 8, 15, 16, 17, 255, 256]), ("9runs", [257, 1, 7, 8, 15, 16, 17, 513, 3]),
                ("17runs", [1, 7, 8, 15, 16, 17, 255, 256, 257, 2, 3, 4, 5, 6, 9, 10, 11])]
    elif log_m <= 16:
        out = [("run%d" % c, [c]) for c in (1, 8, 17, 256, 513)]
        out += [("8runs", [1, 7, 8, 15, 16, 17, 255, 256]), ("9runs", [257, 1, 7, 8, 15, 16, 17, 9, 3]),
                ("17runs", [1, 7, 8, 15, 16, 17, 2, 3, 4, 5, 6, 9, 10, 11, 12, 13, 14])]
    else:
        out = [("run17", [17]), ("run257", [257]), ("9runs", [1, 7, 8, 15, 16, 17, 2, 3, 9]),
               ("17runs", [1, 7, 8, 15, 16, 17, 2, 3, 4, 5, 6, 9, 10, 11, 12, 13, 14])]
    return out


def _check_rows(log_m):
    m = 1 << log_m
    if log_m <= 13:
        return np.arange(m)
    rows = {0, m - 1}
    for b in range(256, (1 << 13) + 1, 256):
        rows |= {b - 1, b}
    rows |= set(np.random.default_rng(log_m).integers(0, m, 2048).tolist())
    return np.array(sorted(rows))


def _place(ctx, cols, counts, merged):
    """upload the logical columns (T, M) into one device buffer; -> (matrix pointers, widths).  Separate runs are laid out in
    decreasing address order (no two runs continue each other); merged ones are adjacent in increasing order, and
    deep_quotient_groups_m must join them into one run."""
    t, m = cols.shape
    starts = np.cumsum([0] + counts)
    if merged:
        d = ctx.to_device(cols)
        return d, [d.ptr + 4 * m * int(s) for s in starts[:-1]], counts
    phys = np.empty_like(cols)
    offs = []
    for i, c in enumerate(counts):
        off = t - int(starts[i + 1])
        phys[off:off + c] = cols[starts[i]:starts[i + 1]]
        offs.append(off)
    d = ctx.to_device(phys)
    return d, [d.ptr + 4 * m * o for o in offs], counts


def _deep_expected(cols, rows, log_m, shift, zeta, gamma, ys):
    gp = ref.gamma_powers(gamma, cols.shape[0])
    ysum = ref.ZERO
    for g, y in zip(gp, ys):
        ysum = ref.e4_add(ysum, ref.e4_mul(g, ref.e4(y)))
    xs = ref.domain_np(log_m, shift, bit_reversed=True)[rows]
    return ref.deep_rows_np(cols[:, rows], gp, ysum, xs, zeta).T


def _deep(ctx, ptrs, widths, log_m, shift, zeta, gamma, ys):
    m = 1 << log_m
    d_ys = ctx.to_device(np.asarray(ys, dtype=np.uint32).reshape(-1, 4))
    d_out = _guarded_out(ctx, 4 * m)
    before = ctx.launch_count()
    ctx.deep_quotient(ptrs, widths, log_m, shift, zeta, gamma, d_ys.ptr, d_out.ptr)
    launches = ctx.launch_count() - before
    raw = d_out.download(4 * m + 16)
    assert (raw[4 * m:] == 0xFFFFFFFF).all(), "pb_deep_quotient wrote past d_out[2^log_m]"
    return raw[:4 * m].reshape(m, 4), launches


@pytest.mark.parametrize("log_m", DQ_LOGS)
def test_deep_quotient_layouts(ctx, log_m):
    rng = np.random.default_rng(300 + log_m)
    m = 1 << log_m
    rows = _check_rows(log_m)
    zetas = [("ext4", tuple(int(x) for x in rng.integers(0, P, 4))), ("base", (int(rng.integers(0, P)), 0, 0, 0)),
             ("limb3", (0, 0, 0, int(rng.integers(1, P)))), ("H", (ref.domain_point(1, log_m, 1), 0, 0, 0))]
    shifts = [31, 1234567, P - 1, 31]
    for li, (name, counts) in enumerate(_layouts(log_m)):
        t = sum(counts)
        cols = rand_field(rng, (t, m))
        cols[0, :] = P - 1
        ys = rand_field(rng, (t, 4))
        shift = shifts[li % len(shifts)]
        zname, zeta = zetas[li % len(zetas)]
        if zname == "base" or zname == "H":
            if shift == P - 1 or ref.in_coset(zeta, shift, log_m):     # -H' = H' contains H's points: a non-member instead
                zeta = (ref.domain_point(shift, log_m + 1, 1), 0, 0, 0)
        assert not ref.in_coset(zeta, shift, log_m)
        gset = GAMMAS if li == 0 else [GAMMAS[li % len(GAMMAS)]]
        for merged in ((False, True) if len(counts) > 1 else (False,)):
            d, ptrs, widths = _place(ctx, cols, counts, merged)
            for gname, gamma in gset:
                got, launches = _deep(ctx, ptrs, widths, log_m, shift, zeta, gamma, ys)
                assert launches == (1 if merged else (len(counts) + 7) // 8), (name, merged, launches)
                exp = _deep_expected(cols, rows, log_m, shift, zeta, gamma, ys)
                bad = np.nonzero((got[rows] != _monty(exp)).any(axis=1))[0]
                assert bad.size == 0, (name, merged, gname, zname, shift, rows[bad[:8]].tolist())
            d.free()


@pytest.mark.parametrize("log_m", DQ_LOGS)
def test_deep_quotient_true_openings_fold_to_a_constant(ctx, log_m):
    """columns of degree < M/2 opened at their true values: the reduced opening has degree < M/2 - 1, so folding it down to
    length 2 gives a constant; every row of the codeword counts towards that"""
    rng = np.random.default_rng(400 + log_m)
    m = 1 << log_m
    counts = [1, 7, 8, 15, 16, 17, 2, 3, 1] if log_m > 2 else [1, 2]
    shift = 31
    deg = max(1, m // 2)
    terms = [[(0, int(rng.integers(0, P))), (deg - 1, P - 1)] + [(int(k), int(rng.integers(0, P))) for k in rng.integers(0, deg, 2)]
             for _ in range(sum(counts))]
    cols = np.stack([ref.sparse_codeword(t, log_m, shift, bit_reversed=True)[0] for t in terms]).astype(np.uint32)
    zeta = tuple(int(x) for x in rng.integers(0, P, 4))
    ys = [ref.eval_sparse(t, zeta) for t in terms]
    gamma = tuple(int(x) for x in rng.integers(0, P, 4))
    d, ptrs, widths = _place(ctx, cols, counts, False)
    got, _ = _deep(ctx, ptrs, widths, log_m, shift, zeta, gamma, ys)
    rows = _check_rows(log_m)
    assert (got[rows] == _monty(_deep_expected(cols, rows, log_m, shift, zeta, gamma, ys))).all()
    # fold the whole codeword down to length 2
    cur = _raw_upload(ctx, got)
    s = shift
    for log_len in range(log_m, 1, -1):
        beta = tuple(int(x) for x in rng.integers(0, P, 4))
        nxt = ctx.alloc(16 << (log_len - 1))
        ctx.fri_fold(cur.ptr, log_len, s, beta, nxt.ptr)
        cur, s = nxt, s * s % P
    fin = cur.download(8).reshape(2, 4)
    assert (fin[0] == fin[1]).all(), "the reduced opening of true openings is not low-degree"


@pytest.mark.parametrize("log_m", [1, 7, 13])
def test_deep_quotient_refuses_zeta_on_the_lde_domain(ctx, log_m):
    """x_r - zeta = 0 at one row: PB_ERR_UNSUPPORTED before any kernel is launched, and d_out untouched"""
    from powdr_b200.capi import PbError
    rng = np.random.default_rng(500 + log_m)
    m = 1 << log_m
    cols = rand_field(rng, (9, m))
    d, ptrs, widths = _place(ctx, cols, [4, 5], False)
    d_ys = ctx.to_device(rand_field(rng, (9, 4)))
    d_out = _guarded_out(ctx, 4 * m)
    for shift in (31, P - 1, 1234567):
        for r in sorted({0, 1, m // 2, m - 1}):
            zeta = (ref.domain_point(shift, log_m, r), 0, 0, 0)
            before = ctx.launch_count()
            with pytest.raises(PbError) as e:
                ctx.deep_quotient(ptrs, widths, log_m, shift, zeta, (5, 6, 7, 8), d_ys.ptr, d_out.ptr)
            assert e.value.code == -2 and ctx.launch_count() == before, (shift, r)
    assert (d_out.download(4 * m + 16) == 0xFFFFFFFF).all()


# ---------------------------------------------------------------- pb_fri_fold
BETAS = [("0", ref.ZERO), ("1", ref.ONE), ("p-1", (P - 1, 0, 0, 0)), ("base", (555555555, 0, 0, 0)), ("ext4", (P - 2, 3, P - 4, 5))]


def _fold_terms(log_len, rng, n_terms=4):
    n = 1 << log_len
    t = [(0, (1, 2, 3, 4)), (n - 1, tuple(int(x) for x in rng.integers(0, P, 4))), (1, (P - 1,) * 4), (int(rng.integers(0, n)), 7)]
    return t[:n_terms]


def _fold(ctx, d_in, log_len, shift, beta):
    half = 1 << (log_len - 1)
    d_out = _guarded_out(ctx, 4 * half)
    ctx.fri_fold(d_in.ptr, log_len, shift, beta, d_out.ptr)
    raw = d_out.download(4 * half + 16)
    assert (raw[4 * half:] == 0xFFFFFFFF).all(), "pb_fri_fold wrote past d_out[len/2]"
    return raw[:4 * half].reshape(half, 4)


def _fold_expected(terms, log_len, shift, beta):
    return _monty(ref.sparse_codeword(ref.fold_sparse(terms, beta), log_len - 1, shift * shift % P, bit_reversed=True).T)


@pytest.mark.parametrize("log_len", list(range(1, 26)))
def test_fri_fold(ctx, log_len):
    rng = np.random.default_rng(600 + log_len)
    shifts = [1, 31, P - 1, pow(31, 1 << (1 + log_len % 5), P)]
    big = log_len >= 22          # the host reference takes seconds per codeword here: one shift, one beta
    if big:
        shifts = [shifts[1 + log_len % 2 * 2]]
    terms = _fold_terms(log_len, rng, 3 if big else 4)
    for si, shift in enumerate(shifts):
        d_in = _raw_upload(ctx, _monty(ref.sparse_codeword(terms, log_len, shift, bit_reversed=True).T))
        betas = [BETAS[4]] if big else BETAS if si == 0 else [BETAS[(log_len + si) % len(BETAS)]]
        for bname, beta in betas:
            got = _fold(ctx, d_in, log_len, shift, beta)
            assert (got == _fold_expected(terms, log_len, shift, beta)).all(), (shift, bname)
        d_in.free()
    if log_len <= 20:
        full = _raw_upload(ctx, _monty(np.full((1 << log_len, 4), P - 1)))
        assert (_fold(ctx, full, log_len, 31, BETAS[4][1]) == _monty([P - 1])).all()


def test_fri_fold_chain_ends_in_the_closed_form_constant(ctx):
    rng = np.random.default_rng(700)
    log_len = 20
    half = 1 << (log_len - 1)
    terms = [(0, (9, 8, 7, 6)), (half - 1, tuple(int(x) for x in rng.integers(0, P, 4))), (1, (P - 1, 0, 0, 1)),
             (int(rng.integers(0, half)), (5, 0, 0, 0))]
    cur = _raw_upload(ctx, _monty(ref.sparse_codeword(terms, log_len, 31, bit_reversed=True).T))
    s = 31
    for ll in range(log_len, 1, -1):
        beta = tuple(int(x) for x in rng.integers(0, P, 4))
        terms = ref.fold_sparse(terms, beta)
        nxt = ctx.alloc(16 << (ll - 1))
        ctx.fri_fold(cur.ptr, ll, s, beta, nxt.ptr)
        cur, s = nxt, s * s % P
    assert [k for k, _ in terms] == [0]
    assert (cur.download(8).reshape(2, 4) == _monty([terms[0][1], terms[0][1]])).all()


def test_fold_table_cache_large_first_and_small_first(ctx):
    """get_fold_table keeps the longest table and serves shorter folds from its prefix; a context that folds short lengths
    first rebuilds it for a longer one.  Both orders give the same words."""
    import powdr_b200
    rng = np.random.default_rng(800)
    lens = [25, 1, 2, 3, 9, 10, 17]
    cases = {}
    for ll in lens:
        terms = _fold_terms(ll, rng, 3)
        beta = tuple(int(x) for x in rng.integers(0, P, 4))
        cases[ll] = (terms, beta, _raw_upload(ctx, _monty(ref.sparse_codeword(terms, ll, 31, bit_reversed=True).T)))

    def run(c, order):
        out = {}
        for ll in order:
            terms, beta, d_in = cases[ll]
            d_out = c.alloc(16 << (ll - 1))
            c.fri_fold(d_in.ptr, ll, 31, beta, d_out.ptr)
            out[ll] = d_out.download((1 << (ll - 1), 4))
        return out
    a = run(ctx, lens)                                   # 2^25 first: the short folds read the prefix of its table
    fresh = powdr_b200.Context(0)
    try:
        b = run(fresh, lens[1:] + [25] + lens[1:])       # short first, then the table is rebuilt for 2^25
    finally:
        fresh.close()
    for ll in lens:
        terms, beta, _ = cases[ll]
        assert (a[ll] == b[ll]).all() and (a[ll] == _fold_expected(terms, ll, 31, beta)).all(), ll
