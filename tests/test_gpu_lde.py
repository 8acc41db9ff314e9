"""Coset LDE (pb_lde_batch, pb_lde_shard) against the scalar oracle, every output word, at every pass geometry (1 <= log_n <= 24:
nttf::transposed_kernel alone up to 2^10, nttf::strided_kernel / transposed_kernel for (n_hi, n_lo) = (5,6) ... (12,12) above,
and the TMA-staged transposed passes at n_lo = 10), with more than one coset, several column batches, twiddle-cache eviction,
words at the edges of the lazy [0, 2p) arithmetic, and the row-sharded LDE.

Device words are compared raw (Montgomery form) with the oracle's LDE converted to Montgomery form, so a kernel that leaves a
word unreduced fails too.  Every output buffer starts as SENTINEL, which is not a valid Montgomery word, so a row the kernel
never writes cannot match by accident.

The oracle runs one column per core.  LdeRefs computes each reference once per module, independent references concurrently,
and serves a smaller blow-up from a larger one (see LdeRefs)."""
import os
import threading
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from util import P, bitrev, rand_field

gpu = pytest.mark.gpu

R_MOD_P = (1 << 32) % P
R_INV = pow(1 << 32, -1, P)
SENTINEL = 0xFFFFFFFF


def mont(a):
    return ((np.asarray(a, dtype=np.uint32).astype(np.uint64) * np.uint64(R_MOD_P)) % np.uint64(P)).astype(np.uint32)


def from_mont(a):
    return ((np.asarray(a, dtype=np.uint32).astype(np.uint64) * np.uint64(R_INV)) % np.uint64(P)).astype(np.uint32)


def root_of_unity(log_n):
    return pow(31, (P - 1) >> log_n, P)


def quotient_shift(log_n):
    """w_{2N}^{-1}: the shift of the second quotient chunk (quotient_chunk_shift in segment.inl); the first one's is 1"""
    return pow(root_of_unity(log_n + 1), P - 2, P)


def random_shift(log_n):
    return int(np.random.default_rng(7000 + log_n).integers(2, P))


def n_lo_of(log_n):
    """low split of the pass geometry, as nttf::n_lo_of in ntt_fast.cuh: K2 blocks are 2^n_lo positions, K1/K3 lanes run over
    k mod 2^n_lo"""
    return log_n if log_n <= 10 else (log_n + 1) // 2


# ---------------------------------------------------------------- comparison
def mismatches(got, exp, log_n, log_blowup, row0=0, limit=6):
    """-> (number of differing words, the first `limit` of them decoded).  got / exp: (width, rows) words of rows [row0, row0 + rows)
    of an LDE with 2^log_blowup cosets.  Row r holds coset c = bitrev_b(r >> n) at natural index k = bitrev_n(r & (N - 1))."""
    diff = got != exp
    count = int(np.count_nonzero(diff))
    flat, rows = diff.ravel(), got.shape[1]
    n_lo = n_lo_of(log_n)
    first, i = [], 0
    while len(first) < min(limit, count):
        i += int(np.argmax(flat[i:]))
        col, r = divmod(i, rows)
        row = row0 + r
        k = bitrev(row & ((1 << log_n) - 1), log_n)
        first.append(dict(col=col, row=row, coset=bitrev(row >> log_n, log_blowup), k=k, k_lo=k & ((1 << n_lo) - 1), k_hi=k >> n_lo,
                          got=int(got[col, r]), exp=int(exp[col, r])))
        i += 1
    return count, first


def assert_lde_equal(got, exp, log_n, log_blowup, row0=0, what="LDE"):
    assert got.shape == exp.shape, (got.shape, exp.shape)
    count, first = mismatches(got, exp, log_n, log_blowup, row0)
    if not count:
        return
    lines = ["%s (log_n %d, log_blowup %d): %d of %d words differ, %d of them still %#x (never written); n_lo = %d"
             % (what, log_n, log_blowup, count, got.size, int(np.count_nonzero((got == SENTINEL) & (exp != SENTINEL))), SENTINEL,
                n_lo_of(log_n))]
    for m in first:
        lines.append("  col {col} row {row}: coset {coset}, k {k} (k mod 2^n_lo = {k_lo}, k >> n_lo = {k_hi}): got {got:#010x}, "
                     "expected {exp:#010x}".format(**m))
    raise AssertionError("\n".join(lines))


# ---------------------------------------------------------------- oracle references
class LdeRefs:
    """Oracle LDEs in Montgomery form, keyed by (seed, log_n, width, log_blowup, shift); the trace is rand_field(seed).

    Rows are bit-reversed over the whole coset domain (row bitrev_{n+b}(j) holds f(shift w_{N 2^b}^j)), so the LDE with 2^b cosets
    is the first N 2^b rows of the one with 2^3 cosets of the same trace and shift: one oracle call serves every blow-up up to its
    own.  get(key, plan) computes the missing references of `plan` together with `key`, concurrently (ctypes releases the GIL)."""

    def __init__(self, orc):
        self.orc, self._traces, self._ldes = orc, {}, {}

    def trace(self, seed, log_n, width):
        k = (seed, log_n, width)
        if k not in self._traces:
            self._traces[k] = rand_field(np.random.default_rng(seed), (width, 1 << log_n))
        return self._traces[k]

    def _cached(self, key):
        seed, log_n, width, log_blowup, shift = key
        for b in range(log_blowup, 4):
            hit = self._ldes.get((seed, log_n, width, b, shift))
            if hit is not None:
                return hit[:, :(1 << log_n) << log_blowup]
        return None

    def _compute(self, key):
        seed, log_n, width, log_blowup, shift = key
        return mont(self.orc.lde_batch(self.trace(seed, log_n, width), log_blowup, shift))

    def get(self, key, plan=()):
        got = self._cached(key)
        if got is not None:
            return got
        todo = [k for k in plan if self._cached(k) is None]
        covered = any(k[:3] == key[:3] and k[4] == key[4] and k[3] >= key[3] for k in todo)
        todo += [] if covered else [key]
        for k in todo:
            self.trace(*k[:3])
        with ThreadPoolExecutor(min(len(todo), os.cpu_count() or 1)) as ex:
            for k, v in zip(todo, ex.map(self._compute, todo)):
                self._ldes[k] = v
        return self._cached(key)


@pytest.fixture(scope="module")
def refs(orc):
    return LdeRefs(orc)


# the geometry tests' trace at each size, and the references they take of it
SMALL_SIZES = list(range(1, 16))        # n_hi = 0 up to 2^10, then (n_hi, n_lo) = (5,6) ... (7,8); every blow-up
GEOM_SIZES = list(range(16, 25))
BLOWUP_SIZES = [16, 19, 20, 24]         # n_lo = 8, 10 (TMA forward pass), 10 (TMA), 12


def geom_width(log_n):
    """up to 2^10 a column is one transposed block: 21 blocks leave 5 of the second CTA's 16 lanes live"""
    return 21 if log_n <= 10 else 3 if log_n <= 21 else 2 if log_n <= 23 else 1


def geom_shifts(log_n):
    return [31, quotient_shift(log_n), random_shift(log_n)]


def geom_key(log_n, log_blowup, shift):
    return (log_n, log_n, geom_width(log_n), log_blowup, shift)


def geom_ref(refs, log_n, log_blowup, shift):
    """the first request at a size computes all of that size's references: one per shift, at the largest blow-up asked for"""
    def top(s):
        return 3 if log_n in SMALL_SIZES or (log_n in BLOWUP_SIZES and s != quotient_shift(log_n)) else 1
    return refs.get(geom_key(log_n, log_blowup, shift), [geom_key(log_n, top(s), s) for s in geom_shifts(log_n)])


def shift_of(kind, log_n):
    return {"31": 31, "quotient": quotient_shift(log_n), "random": random_shift(log_n)}[kind]


# ---------------------------------------------------------------- device calls
def sentinel_buffer(ctx, words):
    return ctx.alloc(4 * words).upload(np.full(words, SENTINEL, dtype=np.uint32))


def run_lde(ctx, words, log_blowup, shift):
    """pb_lde_batch over Montgomery words (width, N) -> raw output words (width, N 2^log_blowup); the input must come back unchanged"""
    width, n = words.shape
    d_in = ctx.to_device(words, monty=False)
    d_out = sentinel_buffer(ctx, width * (n << log_blowup))
    ctx.lde_batch(d_in.ptr, n.bit_length() - 1, width, d_out.ptr, log_blowup, shift)
    got = d_out.download((width, n << log_blowup))
    assert (d_in.download(words.shape) == words).all(), "pb_lde_batch changed its input"
    d_in.free()
    d_out.free()
    return got


def check_geom(ctx, refs, log_n, log_blowup, shift, what):
    exp = geom_ref(refs, log_n, log_blowup, shift)
    got = run_lde(ctx, mont(refs.trace(*geom_key(log_n, log_blowup, shift)[:3])), log_blowup, shift)
    assert_lde_equal(got, exp, log_n, log_blowup, what=what)


# ---------------------------------------------------------------- the helper itself (CPU)
def test_mismatch_report_names_column_coset_and_index(orc):
    log_n, log_blowup, width = 12, 2, 3
    n_lo = n_lo_of(log_n)
    exp = mont(orc.lde_batch(rand_field(np.random.default_rng(1), (width, 1 << log_n)), log_blowup, 31))
    c, k = 1, 5 + (3 << n_lo)
    row = (bitrev(c, log_blowup) << log_n) + bitrev(k, log_n)
    got = exp.copy()
    got[2, row] ^= 1
    count, first = mismatches(got, exp, log_n, log_blowup)
    assert count == 1
    assert first == [dict(col=2, row=row, coset=c, k=k, k_lo=5, k_hi=3, got=int(got[2, row]), exp=int(exp[2, row]))]
    with pytest.raises(AssertionError, match="1 of %d words differ" % exp.size) as e:
        assert_lde_equal(got, exp, log_n, log_blowup)
    assert "col 2 row %d: coset 1, k %d (k mod 2^n_lo = 5, k >> n_lo = 3)" % (row, k) in str(e.value)
    # the same word as part of a row block that starts at row0
    count, first = mismatches(got[:, row - 7:], exp[:, row - 7:], log_n, log_blowup, row0=row - 7)
    assert count == 1 and (first[0]["col"], first[0]["coset"], first[0]["k"]) == (2, c, k)
    assert_lde_equal(exp, exp, log_n, log_blowup)


def test_reference_identities(orc):
    """what LdeRefs and the cache-eviction test derive from one oracle call: the 2^b-coset LDE is the first N 2^b rows of the
    8-coset one, and shift -s swaps rows 2i and 2i + 1"""
    log_n, s = 7, random_shift(7)
    trace = rand_field(np.random.default_rng(2), (2, 1 << log_n))
    top = orc.lde_batch(trace, 3, s)
    for b in (1, 2):
        assert (orc.lde_batch(trace, b, s) == top[:, :(1 << log_n) << b]).all()
    assert (orc.lde_batch(trace, 3, P - s) == top.reshape(2, -1, 2)[:, :, ::-1].reshape(top.shape)).all()


# ---------------------------------------------------------------- 1. every specialised geometry, blow-up 1
@gpu
@pytest.mark.parametrize("shift_kind", ["31", "quotient", "random"])
@pytest.mark.parametrize("log_n", GEOM_SIZES)
def test_lde_every_specialised_geometry_matches_oracle(ctx, refs, log_n, shift_kind):
    """(n_hi, n_lo) = (8,8) at 2^16 ... (12,12) at 2^24, full output; shifts 31, w_{2N}^{-1} (the prover's second quotient chunk)
    and a random one"""
    shift = shift_of(shift_kind, log_n)
    check_geom(ctx, refs, log_n, 1, shift, "blow-up 1, shift %d" % shift)


@gpu
@pytest.mark.parametrize("shift_kind", ["31", "quotient", "random"])
@pytest.mark.parametrize("log_n", SMALL_SIZES)
def test_lde_small_geometries_match_oracle(ctx, refs, log_n, shift_kind):
    """2^1 ... 2^10: one transposed pass each way, then the bit-reversed store; 2^11 ... 2^15: (n_hi, n_lo) = (5,6) ... (7,8).
    Blow-ups 1, 2 and 3, all from one 8-coset reference per shift"""
    shift = shift_of(shift_kind, log_n)
    for log_blowup in (1, 2, 3):
        check_geom(ctx, refs, log_n, log_blowup, shift, "%d cosets, shift %d" % (1 << log_blowup, shift))


# ---------------------------------------------------------------- 2. more than one coset on the specialised passes
@gpu
@pytest.mark.parametrize("shift_kind", ["31", "random"])
@pytest.mark.parametrize("log_blowup", [3, 2])
@pytest.mark.parametrize("log_n", BLOWUP_SIZES)
def test_lde_blowups_on_specialised_passes_match_oracle(ctx, refs, log_n, log_blowup, shift_kind):
    """K2b and K3 with blockIdx.z = coset > 0: the strided forward pass at every size, the TMA forward pass at 2^19 and 2^20"""
    shift = 31 if shift_kind == "31" else random_shift(log_n)
    check_geom(ctx, refs, log_n, log_blowup, shift, "%d cosets, shift %d" % (1 << log_blowup, shift))


# ---------------------------------------------------------------- 3. TMA-staged and LDG/STS-staged transposed passes
@gpu
@pytest.mark.parametrize("tma", [True, False], ids=["tma", "no_tma"])
@pytest.mark.parametrize("log_blowup", [1, 2])
@pytest.mark.parametrize("log_n,width", [(19, 37), (20, 5)])
def test_tma_and_ldg_staged_passes_match_oracle(ctx, refs, monkeypatch, log_n, width, log_blowup, tma):
    """n_lo = 10 runs the two transposed passes on the TMA-staged kernels (ntt_tma.cuh); PB_LDE_NO_TMA=1 selects the LDG/STS-staged
    specialisations.  Both must equal the oracle."""
    if not tma:
        monkeypatch.setenv("PB_LDE_NO_TMA", "1")
    key = (300 + log_n, log_n, width, log_blowup, 31)
    exp = refs.get(key, [key[:3] + (2, 31)])
    got = run_lde(ctx, mont(refs.trace(*key[:3])), log_blowup, 31)
    assert_lde_equal(got, exp, log_n, log_blowup, what="TMA" if tma else "PB_LDE_NO_TMA=1")


# ---------------------------------------------------------------- 4. words at the edges of the lazy arithmetic
def edge_columns(log_n):
    """Montgomery words: constants 0, 1, P-1, P-2 and R mod p (= 1), 0 / P-1 alternating, a P-1 delta at row 0 and one at row N-1,
    and the evaluations of the polynomial whose coefficient words are all P-1 (P - N at row 0, 0 elsewhere)"""
    n = 1 << log_n
    cols = [np.full(n, w, dtype=np.uint32) for w in (0, 1, P - 1, P - 2, R_MOD_P)]
    alt = np.zeros(n, dtype=np.uint32)
    alt[1::2] = P - 1
    d0, d1, coef = np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.uint32)
    d0[0], d1[-1], coef[0] = P - 1, P - 1, P - n
    return np.stack(cols + [alt, d0, d1, coef]), 5


@gpu
@pytest.mark.parametrize("log_n", [16, 20])
def test_lde_at_reduction_edges_matches_oracle(ctx, orc, log_n):
    words, n_const = edge_columns(log_n)
    exp3 = mont(orc.lde_batch(from_mont(words), 3, 31))
    for log_blowup in (1, 3):
        got = run_lde(ctx, words, log_blowup, 31)
        assert_lde_equal(got, exp3[:, :(1 << log_n) << log_blowup], log_n, log_blowup, what="edge columns")
        # a constant polynomial is that constant on every coset: holds whatever the oracle says
        assert (got[:n_const] == words[:n_const, :1]).all()


# ---------------------------------------------------------------- 5. several column batches per call
@gpu
@pytest.mark.parametrize("batch", [1, 3, 5])
@pytest.mark.parametrize("width", [7, 13])
@pytest.mark.parametrize("log_n", [9, 13, 16, 20])
def test_lde_column_batches_match_oracle(ctx, refs, monkeypatch, log_n, width, batch):
    """PB_LDE_BATCH splits one call into ceil(width / batch) equal batches but the last (7 by 3: 3 + 3 + 1; 13 by 5: 5 + 5 + 3);
    4 cosets, so each batch writes its own slice of the output rows as well"""
    monkeypatch.setenv("PB_LDE_BATCH", str(batch))
    key = (500 + log_n, log_n, 13, 2, 31)                       # width 7 is the first 7 columns of the 13-column trace
    exp = refs.get(key)[:width]
    got = run_lde(ctx, mont(refs.trace(*key[:3])[:width]), 2, 31)
    assert_lde_equal(got, exp, log_n, 2, what="PB_LDE_BATCH=%d" % batch)


# ---------------------------------------------------------------- 6. twiddle-cache eviction
def own_context():
    import powdr_b200
    return powdr_b200.Context(0)


@gpu
def test_twiddle_cache_evicts_beyond_64_sets(refs):
    """65 distinct (n, blow-up, shift) sets on a fresh context push the first out of the cache (FIFO over 64 sets); using it
    again rebuilds it"""
    log_n, seed = 16, 600
    keys = [(seed, log_n, 1, 1, 31 + 2 * i) for i in range(65)]
    words = mont(refs.trace(seed, log_n, 1))
    c2 = own_context()
    try:
        for key in keys + keys[:1]:
            got = run_lde(c2, words, 1, key[4])
            assert_lde_equal(got, refs.get(key, keys), log_n, 1, what="shift %d" % key[4])
    finally:
        c2.close()


@gpu
def test_twiddle_cache_evicts_beyond_4_gib(refs):
    """four 2^24-row, 8-coset sets (1.2 GB of tables each) push the cache past 4 GiB and the first set out; using it again
    rebuilds it.  Shift -s evaluates coset row j + N 2^b / 2 where shift s evaluates row j, i.e. it swaps rows 2i and 2i + 1."""
    log_n = 24
    base = [31, random_shift(log_n)]
    sets = [(s, False) for s in base] + [(P - s, True) for s in base]
    words = mont(refs.trace(*geom_key(log_n, 3, 31)[:3]))
    c2 = own_context()
    try:
        for i in [0, 1, 2, 3, 0]:
            shift, negated = sets[i]
            exp = geom_ref(refs, log_n, 3, base[i % 2])
            if negated:
                exp = exp.reshape(exp.shape[0], -1, 2)[:, :, ::-1].reshape(exp.shape)
            got = run_lde(c2, words, 3, shift)
            assert_lde_equal(got, exp, log_n, 3, what="set %d, shift %d" % (i, shift))
    finally:
        c2.close()


# ---------------------------------------------------------------- 7. the row-sharded LDE
@gpu
@pytest.mark.parametrize("shift_kind", ["31", "quotient"])
@pytest.mark.parametrize("world", [2, 8])
@pytest.mark.parametrize("log_n", [11, 16, 20, 24])
def test_lde_shard_matches_oracle(ctx, refs, log_n, world, shift_kind):
    """pb_lde_shard block b = rows [b Ms, (b + 1) Ms) of the 2-coset LDE, Ms = 2N / world; its forward pass has 2^(n + 1 - g) rows,
    g = log2(world): 2^9 (one transposed pass, then the bit-reversed store), 2^11, 2^14, 2^16, 2^18, 2^20, 2^22 and 2^24"""
    shift = 31 if shift_kind == "31" else quotient_shift(log_n)
    width = geom_width(log_n)
    exp = geom_ref(refs, log_n, 1, shift)
    words = mont(refs.trace(*geom_key(log_n, 1, shift)[:3]))
    ms = (2 << log_n) // world
    d_in = ctx.to_device(words, monty=False)
    d_blk = ctx.alloc(4 * width * ms)
    sentinel = np.full(width * ms, SENTINEL, dtype=np.uint32)
    for blk in range(world):
        d_blk.upload(sentinel)
        ctx.lde_shard(d_in.ptr, log_n, width, world, blk, d_blk.ptr, shift)
        got = d_blk.download((width, ms))
        assert_lde_equal(got, exp[:, blk * ms:(blk + 1) * ms], log_n, 1, row0=blk * ms, what="shard %d of %d" % (blk, world))
    assert (d_in.download(words.shape) == words).all(), "pb_lde_shard changed its input"


# ---------------------------------------------------------------- 8. two GPUs in one process
def device_count():
    import torch
    return torch.cuda.device_count()


@gpu
def test_lde_on_two_devices_in_one_process(refs, monkeypatch):
    """one context per device, each used from its own thread (pb_ctx_create makes its device current for that thread): the
    64 KB+ dynamic shared memory opt-in of the specialised and TMA kernels must hold on both devices"""
    if device_count() < 2:
        pytest.skip("needs two visible CUDA devices")
    import powdr_b200
    log_n = 20
    exp = geom_ref(refs, log_n, 2, 31)
    words = mont(refs.trace(*geom_key(log_n, 2, 31)[:3]))

    def on_device(dev, out):
        c = None
        try:
            c = powdr_b200.Context(dev)
            out[dev] = run_lde(c, words, 2, 31)
        except BaseException as e:          # noqa: BLE001
            out[dev] = e
        finally:
            if c is not None:
                c.close()

    for tma in (True, False):
        if not tma:
            monkeypatch.setenv("PB_LDE_NO_TMA", "1")
        out = {}
        for dev in (0, 1):
            t = threading.Thread(target=on_device, args=(dev, out))
            t.start()
            t.join()
        for dev in (0, 1):
            if isinstance(out[dev], BaseException):
                raise out[dev]
            assert_lde_equal(out[dev], exp, log_n, 2, what="device %d, %s" % (dev, "TMA" if tma else "PB_LDE_NO_TMA=1"))
