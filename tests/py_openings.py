"""Plain reference for the opening phase: the openings f(zeta), the DEEP reduced opening and the arity-2 FRI fold, over
BabyBear and its quartic extension F_p[x]/(x^4 - 11).

Field arithmetic is on Python integers (scalars) or on uint64 numpy arrays reduced mod p after every product (whole
codewords); no Montgomery form, and nothing is imported from the oracle or the library.  Ext4 elements are 4-tuples of
canonical limbs, lowest degree first.

A sparse polynomial is a list of (k, c) terms, f(x) = sum_t c_t x^k_t, c_t an int (base field) or an Ext4 tuple.  Its value
at any point is exact in closed form, so it checks an opening, a reduced opening or a fold at any height.
"""
import numpy as np

P = 2013265921
W = 11                  # x^4 = W
GEN = 31                # generator of F_p^*


# ---------------------------------------------------------------- base field and Ext4, Python integers
def e4(a):
    """int or 4-sequence -> canonical Ext4 tuple"""
    if isinstance(a, (int, np.integer)):
        return (int(a) % P, 0, 0, 0)
    return tuple(int(x) % P for x in a)


ZERO, ONE = (0, 0, 0, 0), (1, 0, 0, 0)


def e4_add(a, b):
    return tuple((x + y) % P for x, y in zip(a, b))


def e4_sub(a, b):
    return tuple((x - y) % P for x, y in zip(a, b))


def e4_scale(a, s):
    return tuple(x * s % P for x in a)


def e4_mul(a, b):
    t = [0] * 7
    for i in range(4):
        for j in range(4):
            t[i + j] += a[i] * b[j]
    return ((t[0] + W * t[4]) % P, (t[1] + W * t[5]) % P, (t[2] + W * t[6]) % P, t[3] % P)


def e4_pow(a, e):
    r = ONE
    while e:
        if e & 1:
            r = e4_mul(r, a)
        a = e4_mul(a, a)
        e >>= 1
    return r


def e4_inv(a):
    """a^(p^4 - 2): the inverse of a non-zero element (0 for 0)"""
    return e4_pow(a, P ** 4 - 2)


def is_base(a):
    return a[1] == a[2] == a[3] == 0


def root_of_unity(log_n):
    """generator of the order-2^log_n subgroup: 31^((p-1)/2^log_n)"""
    return pow(GEN, (P - 1) >> log_n, P)


def bitrev(i, bits):
    r = 0
    for _ in range(bits):
        r = (r << 1) | (i & 1)
        i >>= 1
    return r


def domain_point(shift, log_n, i):
    """shift * w_N^i"""
    return shift * pow(root_of_unity(log_n), i, P) % P


def in_coset(z, shift, log_n):
    """z lies on shift*H, |H| = 2^log_n (only base-field points can)"""
    z = e4(z)
    return is_base(z) and z[0] != 0 and pow(z[0] * pow(shift, P - 2, P) % P, 1 << log_n, P) == 1


SHIFTS = (1, GEN, P - 1, 1234567)


def zeta_cases(log_n, shift, rng):
    """(name, zeta, row or None): the opening points where a formula over the domain can go wrong.  `row` is set for the
    points shift*w^row of the domain itself, where f(zeta) is the column's value at that row."""
    n = 1 << log_n
    r = lambda: int(rng.integers(0, P))
    cases = [("ext4", (r(), r(), r(), r()), None), ("base", (r(), 0, 0, 0), None), ("zero", ZERO, None), ("one", ONE, None),
             ("all_p-1", (P - 1,) * 4, None)]
    for pos in (1, 2, 3):
        z = [0, 0, 0, 0]
        z[pos] = r() or 1
        cases.append(("limb%d" % pos, tuple(z), None))
    for i in sorted({0, 1, n // 2, n - 1}):
        cases.append(("row%d" % i, (domain_point(shift, log_n, i), 0, 0, 0), i))
    out = []
    for name, z, row in cases:
        if row is None and in_coset(z, shift, log_n):     # 1 with shift 1 (or p-1) is the domain's row 0 (or N/2)
            row = next(i for i in (0, n // 2) if domain_point(shift, log_n, i) == z[0])
        out.append((name, z, row))
    return out


# ---------------------------------------------------------------- openings
def interpolate(col):
    """coefficients of the polynomial of degree < N through col[i] at w_N^i (naive inverse DFT, exact)"""
    v = np.asarray(col, dtype=np.uint64) % np.uint64(P)
    n = v.size
    log_n = n.bit_length() - 1
    assert n == 1 << log_n and n <= 1 << 12
    w_inv = pow(root_of_unity(log_n), P - 2, P)
    pw = np.array([pow(w_inv, e, P) for e in range(n)], dtype=np.uint64)
    ik = (np.arange(n, dtype=np.int64)[:, None] * np.arange(n, dtype=np.int64)[None, :]) % n
    s = ((pw[ik] * v[None, :]) % np.uint64(P)).sum(axis=1) % np.uint64(P)
    n_inv = pow(n, P - 2, P)
    return [int(x) * n_inv % P for x in s]


def horner(coefs, z):
    acc = ZERO
    for c in reversed(coefs):
        acc = e4_add(e4_mul(acc, z), e4(c))
    return acc


def eval_dense(col, shift, zeta):
    """f(zeta) for a column of evaluations over shift*H (natural order): interpolate g(y) = f(shift*y), then g(zeta/shift)"""
    z = e4_scale(e4(zeta), pow(shift, P - 2, P))
    return horner(interpolate(col), z)


def eval_sparse(terms, z):
    """sum_t c_t z^k_t"""
    acc = ZERO
    for k, c in terms:
        acc = e4_add(acc, e4_mul(e4(c), e4_pow(e4(z), k)))
    return acc


def lagrange_at(log_n, shift, s, zeta):
    """L_s(zeta): the polynomial of degree < N that is 1 at shift*w^s and 0 elsewhere on shift*H, as the geometric sum
    (1/N) sum_{k<N} u^k = (u^N - 1) / (N (u - 1)), u = zeta / (shift*w^s)"""
    n = 1 << log_n
    u = e4_scale(e4(zeta), pow(domain_point(shift, log_n, s), P - 2, P))
    if u == ONE:
        return ONE
    num = e4_sub(e4_pow(u, n), ONE)
    return e4_mul(e4_scale(num, pow(n, P - 2, P)), e4_inv(e4_sub(u, ONE)))


def spike_rows(log_n):
    """rows of a single p-1 spike: the ends of the first 256-row CTA and of the first 2^15-row split, and the last row"""
    return sorted(s for s in {0, 255, 256, (1 << 15) - 1, 1 << 15, (1 << log_n) - 1} if s < 1 << log_n)


def edge_columns(log_n, rng):
    """(columns (width, N) uint32 over H, expected(shift, zeta) -> [width] Ext4 f_k(zeta) for the columns read as evaluations
    over shift*H): two sparse polynomials, all p-1, all 0, 0/p-1 alternating, and a p-1 spike at each of spike_rows"""
    n = 1 << log_n
    sa = [(0, int(rng.integers(0, P))), (1, P - 1), (n - 1, int(rng.integers(0, P)))] + [(int(k), int(rng.integers(0, P))) for k in rng.integers(0, n, 2)]
    sb = [(n // 2, 1), (max(0, n - 2), P - 1)]
    half = (P - 1) * pow(2, P - 2, P) % P
    spikes = spike_rows(log_n)
    mat = np.zeros((5 + len(spikes), n), dtype=np.uint32)
    exps = []
    for c, terms in enumerate((sa, sb)):
        mat[c] = sparse_codeword(terms, log_n, 1)[0]
        exps.append(lambda z, t=terms: eval_sparse(t, z))
    mat[2] = P - 1
    exps.append(lambda z: (P - 1, 0, 0, 0))
    exps.append(lambda z: ZERO)                                             # column 3: all 0
    mat[4, 1::2] = P - 1
    exps.append(lambda z: eval_sparse([(0, half), (n // 2, P - half)], z))      # (p-1)(1 - y^(N/2))/2: y^(N/2) = (-1)^i on H
    for c, s in enumerate(spikes):
        mat[5 + c, s] = P - 1
        exps.append(lambda z, s=s: e4_scale(lagrange_at(log_n, 1, s, z), P - 1))

    def expected(shift, zeta):
        y = e4_scale(e4(zeta), pow(shift, P - 2, P))           # the columns are g(w^i), and f(zeta) = g(zeta / shift)
        return [e(y) for e in exps]
    return mat, expected


# ---------------------------------------------------------------- DEEP reduced opening and FRI fold, one value
def gamma_powers(gamma, n):
    out, cur = [], ONE
    for _ in range(n):
        out.append(cur)
        cur = e4_mul(cur, e4(gamma))
    return out


def deep_row(vals, ys, gamma, x, zeta):
    """sum_j gamma^j (f_j(x) - y_j) / (x - zeta) for base-field f_j(x) = vals[j] at the base-field point x"""
    acc = ZERO
    for g, v, y in zip(gamma_powers(gamma, len(vals)), vals, ys):
        acc = e4_add(acc, e4_mul(g, e4_sub(e4(v), e4(y))))
    return e4_mul(acc, e4_inv(e4_sub(e4(x), e4(zeta))))


def fold_pair(lo, hi, x, beta):
    """(lo + hi)/2 + beta (lo - hi) / (2x), lo = f(x), hi = f(-x)"""
    h = pow(2, P - 2, P)
    s = e4_scale(e4_add(lo, hi), h)
    d = e4_scale(e4_sub(lo, hi), h * pow(x, P - 2, P) % P)
    return e4_add(s, e4_mul(e4(beta), d))


def fold_sparse(terms, beta):
    """f = f_e(x^2) + x f_o(x^2)  ->  f_e + beta f_o, as sparse terms with Ext4 coefficients"""
    out = {}
    for k, c in terms:
        c = e4(c)
        if k & 1:
            k2, c2 = (k - 1) // 2, e4_mul(e4(beta), c)
        else:
            k2, c2 = k // 2, c
        out[k2] = e4_add(out.get(k2, ZERO), c2)
    return sorted(out.items())


# ---------------------------------------------------------------- whole codewords, numpy uint64 (reduced after every product)
_P64 = np.uint64(P)


def geom(r, log_n, bit_reversed=False):
    """[r^i] for i < 2^log_n, or [r^bitrev(i)], by doubling: the second half is the first times r^(2^s) (natural) or
    r^(2^(log_n-1-s)) (bit-reversed, as bitrev(i + 2^s) = bitrev(i) + 2^(log_n-1-s))"""
    a = np.ones(1, dtype=np.uint64)
    for s in range(log_n):
        e = 1 << (log_n - 1 - s if bit_reversed else s)
        a = np.concatenate([a, a * np.uint64(pow(r, e, P)) % _P64])
    return a


def sparse_codeword(terms, log_n, shift, bit_reversed=False):
    """f(shift * w_N^i) (or at i = bitrev(j)) for i < N -> uint64 array (4, N) of Ext4 limbs"""
    w = root_of_unity(log_n)
    out = np.zeros((4, 1 << log_n), dtype=np.uint64)
    for k, c in terms:
        c = e4(c)
        xs = geom(pow(w, k, P), log_n, bit_reversed) * np.uint64(pow(shift, k, P)) % _P64
        for l in range(4):
            if c[l]:
                out[l] = (out[l] + xs * np.uint64(c[l]) % _P64) % _P64
    return out


def domain_np(log_n, shift, bit_reversed=False):
    """the points shift * w_N^i (or at i = bitrev(j)), uint64"""
    return geom(root_of_unity(log_n), log_n, bit_reversed) * np.uint64(shift % P) % _P64


def e4_mul_np(a, b):
    """limb-wise arrays (4, n) x (4, n) -> (4, n), uint64"""
    a = [x.astype(np.uint64) for x in a]
    b = [x.astype(np.uint64) for x in b]
    t = [np.zeros_like(a[0]) for _ in range(7)]
    for i in range(4):
        for j in range(4):
            t[i + j] = (t[i + j] + a[i] * b[j] % _P64) % _P64
    w = np.uint64(W)
    return np.stack([(t[0] + t[4] * w % _P64) % _P64, (t[1] + t[5] * w % _P64) % _P64, (t[2] + t[6] * w % _P64) % _P64, t[3]])


def e4_inv_np(a):
    """a^(p^4 - 2) element-wise, (4, n)"""
    r = np.zeros_like(a, dtype=np.uint64)
    r[0] = 1
    base, e = a.astype(np.uint64), P ** 4 - 2
    while e:
        if e & 1:
            r = e4_mul_np(r, base)
        base = e4_mul_np(base, base)
        e >>= 1
    return r


def deep_rows_np(cols, gammas, ysum, xs, zeta):
    """reduced opening at the rows of `cols` ((n_cols, n) base-field values at the points xs): (sum_j gammas[j] cols[j] - ysum)
    / (xs - zeta) -> (4, n) uint64.  gammas: [n_cols] Ext4; ysum: sum_j gammas[j] y_j"""
    f = np.asarray(cols, dtype=np.uint64)
    num = []
    for l in range(4):
        g = np.array([gm[l] for gm in gammas], dtype=np.uint64)
        # at most 2^22 columns before the uint64 sum of reduced products could overflow
        num.append(((f * g[:, None]) % _P64).sum(axis=0) % _P64)
    num = np.stack(num)
    for l in range(4):
        num[l] = (num[l] + np.uint64((P - ysum[l]) % P)) % _P64
    den = np.stack([(np.asarray(xs, dtype=np.uint64) + np.uint64((P - zeta[0]) % P)) % _P64] +
                   [np.full(len(xs), (P - zeta[l]) % P, dtype=np.uint64) for l in (1, 2, 3)])
    return e4_mul_np(num, e4_inv_np(den))
