"""ORACLE (test infrastructure, not product code): ctypes view of oracle/_build/liborc.so.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may import this.
All values are canonical BabyBear u32; matrices are column-major numpy uint32 arrays of shape (width, height).
"""
import ctypes as C
import os
import subprocess
import numpy as np

_DIR = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_DIR, "_build", "liborc.so")
P = 2013265921
GENERATOR = 31


def build(force=False):
    srcs = [os.path.join(_DIR, f) for f in ("ntt.c", "poseidon2.c", "air.c", "prove.c", "verify.c", "fast.c", "logup.c", "oracle.h", "bb31.h")]
    srcs.append(os.path.join(os.path.dirname(_DIR), "include", "pb_poseidon2_constants.h"))
    if force or not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in srcs):
        subprocess.check_call(["make", "-C", _DIR, "-s"])
    return _SO


class Span(C.Structure):
    _fields_ = [("off", C.c_uint32), ("len", C.c_uint32)]


class OriginalAir(C.Structure):
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("buffer", C.c_void_p), ("row_block_size", C.c_int32)]


class Subst(C.Structure):
    _fields_ = [("air_index", C.c_int32), ("col", C.c_int32), ("row", C.c_int32), ("apc_col", C.c_int32)]


class DerivedSpec(C.Structure):
    _fields_ = [("col_base", C.c_uint64), ("span", Span)]


class Interaction(C.Structure):
    _fields_ = [("bus_id", C.c_uint32), ("num_args", C.c_uint32), ("args_index_off", C.c_uint32)]


class AirC(C.Structure):
    _fields_ = [("bc", C.c_void_p), ("spans", C.c_void_p), ("n_constraints", C.c_size_t),
                ("ibc", C.c_void_p), ("ispans", C.c_void_p), ("ints", C.c_void_p), ("n_ints", C.c_size_t)]


class ParamsC(C.Structure):
    _fields_ = [("n_queries", C.c_uint32), ("pow_bits", C.c_uint32), ("fast", C.c_int), ("cheat_opening", C.c_int)]


class Air:
    """orc_air_t: constraints (bytecode, spans) + bus interactions `bus` = (interactions [(bus_id, num_args, args_index_off)],
    arg_spans [(off, len)], bytecode) as returned by powdr_b200.machine.compile_bus(machine, 1) (column-index convention)."""

    def __init__(self, bc, spans, bus=None):
        self.bc = _u32(bc)
        self.spans = compile_spans(spans)
        self.n_constraints = len(spans)
        ints, isp, ibc = bus if bus else ([], [], [])
        self.ibc = _u32(ibc if len(ibc) else [0])
        self.ispans = compile_spans(isp)
        self.ints = (Interaction * max(1, len(ints)))()
        for i, (b, n, o) in enumerate(ints):
            self.ints[i].bus_id, self.ints[i].num_args, self.ints[i].args_index_off = b, n, o
        self.n_ints = len(ints)
        self.c = AirC(self.bc.ctypes.data, C.addressof(self.spans), self.n_constraints, self.ibc.ctypes.data, C.addressof(self.ispans),
                      C.addressof(self.ints), self.n_ints)

    @property
    def perm_width(self):
        lib().orc_perm_width.restype = C.c_size_t
        return int(lib().orc_perm_width(C.byref(self.c)))


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_SO)
        _lib.orc_eval_expr.restype = C.c_uint32
        _lib.orc_challenger_sample.restype = C.c_uint32
        _lib.orc_num_threads.restype = C.c_int
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _u32(a):
    return np.ascontiguousarray(a, dtype=np.uint32)


def num_threads():
    return lib().orc_num_threads()


def dft_naive(coeffs, shift=1):
    a = _u32(coeffs)
    out = np.empty_like(a)
    lib().orc_dft_naive(_p(a), _p(out), C.c_uint(a.size.bit_length() - 1), C.c_uint32(shift))
    return out


def ntt(a):
    a = _u32(a).copy()
    lib().orc_ntt(_p(a), C.c_uint(a.size.bit_length() - 1))
    return a


def intt(a):
    a = _u32(a).copy()
    lib().orc_intt(_p(a), C.c_uint(a.size.bit_length() - 1))
    return a


def lde_batch(trace, log_blowup=1, shift=GENERATOR):
    """trace: (width, n) column-major -> (width, n << log_blowup), rows bit-reversed."""
    t = _u32(trace)
    w, n = t.shape
    out = np.empty((w, n << log_blowup), dtype=np.uint32)
    lib().orc_lde_batch(_p(t), C.c_uint(n.bit_length() - 1), C.c_size_t(w), C.c_uint(log_blowup), C.c_uint32(shift), _p(out))
    return out


def poseidon2_permute(state):
    s = _u32(state).copy()
    assert s.size == 16
    lib().orc_poseidon2_permute(_p(s))
    return s


def poseidon2_permute_with(state, rc_ext, rc_int, diag):
    s, a, b, c = _u32(state).copy(), _u32(rc_ext), _u32(rc_int), _u32(diag)
    assert s.size == 16 and a.size == 128 and b.size == 13 and c.size == 16
    lib().orc_poseidon2_permute_with(_p(s), _p(a), _p(b), _p(c))
    return s


def set_poseidon2(rc_ext, rc_int, diag):
    """run poseidon2_permute, hash_row, compress, merkle_commit, the challenger, prove and verify (not the AVX-512 fast paths) under
    this instantiation (canonical rc_ext [8][16], rc_int [13], diag [16]) until reset_poseidon2; process-wide"""
    a, b, c = _u32(rc_ext), _u32(rc_int), _u32(diag)
    assert a.size == 128 and b.size == 13 and c.size == 16
    lib().orc_set_poseidon2(_p(a), _p(b), _p(c))


def reset_poseidon2():
    lib().orc_reset_poseidon2()


def hash_row(row):
    r = _u32(row)
    d = np.empty(8, dtype=np.uint32)
    lib().orc_hash_row(_p(r), C.c_size_t(r.size), _p(d))
    return d


def compress(l, r):
    l, r = _u32(l), _u32(r)
    d = np.empty(8, dtype=np.uint32)
    lib().orc_compress(_p(l), _p(r), _p(d))
    return d


def merkle_commit(mats):
    """mats: list of (width_i, h) column-major arrays of equal height -> list of digest layers [(h,8),(h/2,8),...,(1,8)]."""
    mats = [_u32(m) for m in mats]
    h = mats[0].shape[1]
    log_h = h.bit_length() - 1
    ptrs = (C.c_void_p * len(mats))(*[m.ctypes.data for m in mats])
    widths = (C.c_size_t * len(mats))(*[m.shape[0] for m in mats])
    flat = np.empty((2 * h - 1, 8), dtype=np.uint32)
    lib().orc_merkle_commit(ptrs, widths, C.c_size_t(len(mats)), C.c_uint(log_h), _p(flat))
    layers, off, n = [], 0, h
    while n >= 1:
        layers.append(flat[off:off + n])
        off += n
        n >>= 1
    return layers


def compile_spans(spans):
    arr = (Span * max(1, len(spans)))()
    for i, (o, l) in enumerate(spans):
        arr[i].off, arr[i].len = o, l
    return arr


def eval_expr(bc, mat_flat, r):
    bc = _u32(bc)
    m = _u32(mat_flat)
    return lib().orc_eval_expr(_p(bc), C.c_uint32(bc.size), _p(m), C.c_size_t(r))


def constraint_fold(bc, spans, mat, alpha):
    bc, m, al = _u32(bc), _u32(mat), _u32(alpha)
    w, h = m.shape
    out = np.empty((4, h), dtype=np.uint32)
    lib().orc_constraint_fold(_p(bc), compile_spans(spans), C.c_size_t(len(spans)), _p(m), C.c_size_t(h), _p(al), _p(out))
    return out


def quotient(bc, spans, lde, log_n, alpha, shift=GENERATOR):
    bc, m, al = _u32(bc), _u32(lde), _u32(alpha)
    n = 1 << log_n
    out = np.empty((2, 4, n), dtype=np.uint32)
    lib().orc_quotient(_p(bc), compile_spans(spans), C.c_size_t(len(spans)), _p(m), C.c_uint(log_n), C.c_uint(1),
                       C.c_uint32(shift), _p(al), _p(out))
    return out


def eval_at_point(mat, shift, zeta):
    """mat: (width, n) evaluations over shift*H, natural order -> (width, 4) values f(zeta)"""
    m, z = _u32(mat), _u32(zeta)
    w, n = m.shape
    out = np.empty((w, 4), dtype=np.uint32)
    lib().orc_eval_at_point(_p(m), C.c_uint(n.bit_length() - 1), C.c_size_t(w), C.c_uint32(shift), _p(z), _p(out))
    return out


def deep_quotient(mats, shift, zeta, gamma, ys):
    """mats: list of (width_i, m) column-major LDE matrices (bit-reversed rows over shift*H'); ys: (sum width, 4) -> (m, 4).
    ValueError when zeta lies on shift*H'."""
    mats = [_u32(x) for x in mats]
    m = mats[0].shape[1]
    ptrs = (C.c_void_p * len(mats))(*[x.ctypes.data for x in mats])
    widths = (C.c_size_t * len(mats))(*[x.shape[0] for x in mats])
    z, g, y = _u32(zeta), _u32(gamma), _u32(ys)
    out = np.empty((m, 4), dtype=np.uint32)
    if lib().orc_deep_quotient(ptrs, widths, C.c_size_t(len(mats)), C.c_uint(m.bit_length() - 1), C.c_uint32(shift), _p(z), _p(g), _p(y), _p(out)):
        raise ValueError("zeta lies on the LDE domain: the reduced opening has no value at one row")
    return out


def fri_fold(f, shift, beta):
    """f: (len, 4) ext elements, bit-reversed over shift*<w_len> -> (len/2, 4)."""
    f, b = _u32(f), _u32(beta)
    n = f.shape[0]
    out = np.empty((n // 2, 4), dtype=np.uint32)
    lib().orc_fri_fold(_p(f), C.c_uint(n.bit_length() - 1), C.c_uint32(shift), _p(b), _p(out))
    return out


class Challenger:
    class _S(C.Structure):
        _fields_ = [("sponge", C.c_uint32 * 16), ("in_buf", C.c_uint32 * 8), ("n_in", C.c_int),
                    ("out_buf", C.c_uint32 * 8), ("n_out", C.c_int)]

    def __init__(self):
        self.s = Challenger._S()
        lib().orc_challenger_init(C.byref(self.s))

    def observe(self, vals):
        v = _u32(vals)
        lib().orc_challenger_observe(C.byref(self.s), _p(v), C.c_size_t(v.size))

    def sample(self):
        return int(lib().orc_challenger_sample(C.byref(self.s)))

    def sample_ext(self):
        return [self.sample() for _ in range(4)]


def apc_tracegen(H, width, airs, subs, num_calls):
    """airs: list of (col-major array (w,h), row_block_size); subs: list of (air_index, col, row, apc_col)."""
    out = np.full((width, H), 0xDEADBEEF % P, dtype=np.uint32)
    keep = [_u32(a) for a, _ in airs]
    A = (OriginalAir * len(airs))()
    for i, (a, rbs) in enumerate(airs):
        A[i].width, A[i].height, A[i].buffer, A[i].row_block_size = keep[i].shape[0], keep[i].shape[1], keep[i].ctypes.data, rbs
    S = (Subst * max(1, len(subs)))()
    for i, s in enumerate(subs):
        S[i].air_index, S[i].col, S[i].row, S[i].apc_col = s
    lib().orc_apc_tracegen(_p(out), C.c_size_t(H), A, S, C.c_size_t(len(subs)), C.c_int(num_calls))
    return out


def apc_apply_derived(out, num_calls, specs, bc):
    """specs: list of (col_index, off, len); in-place on `out` (width, H)."""
    H = out.shape[1]
    D = (DerivedSpec * max(1, len(specs)))()
    for i, (c, o, l) in enumerate(specs):
        D[i].col_base, D[i].span.off, D[i].span.len = c * H, o, l
    bc = _u32(bc)
    lib().orc_apc_apply_derived_expr(_p(out), C.c_size_t(H), C.c_int(num_calls), D, C.c_size_t(len(specs)), _p(bc))
    return out


def apc_apply_bus(out, num_calls, bc, interactions, arg_spans, var=(3, 1 << 18), tuple2=(7, 256, 2048), bitwise=6):
    bc = _u32(bc)
    I = (Interaction * max(1, len(interactions)))()
    for i, (b, n, o) in enumerate(interactions):
        I[i].bus_id, I[i].num_args, I[i].args_index_off = b, n, o
    var_hist = np.zeros(var[1], dtype=np.uint32)
    t_hist = np.zeros(tuple2[1] * tuple2[2], dtype=np.uint32)
    b_hist = np.zeros(1 << 17, dtype=np.uint32)
    lib().orc_apc_apply_bus(_p(_u32(out)), C.c_int(num_calls), _p(bc), I, C.c_size_t(len(interactions)), compile_spans(arg_spans),
                            C.c_uint32(var[0]), _p(var_hist), C.c_size_t(var[1]), C.c_uint32(tuple2[0]), _p(t_hist),
                            C.c_uint32(tuple2[1]), C.c_uint32(tuple2[2]), C.c_uint32(bitwise), _p(b_hist))
    return var_hist, t_hist, b_hist


def grind(challenger, bits):
    lib().orc_grind.restype = C.c_uint32
    return int(lib().orc_grind(C.byref(challenger.s), C.c_uint(bits)))


def logup_perm_trace(trace, bus, alpha_lu, beta_lu):
    """-> (perm (4*(n_chunks+1), N), cumulative sum [4], chunk_start list)"""
    t = _u32(trace)
    w, n = t.shape
    air = Air([], [], bus)
    cs = np.zeros(air.n_ints + 1, dtype=np.uint32)
    lib().orc_logup_chunks.restype = C.c_int
    ibc, isp, ints = C.c_void_p(air.c.ibc), C.c_void_p(air.c.ispans), C.c_void_p(air.c.ints)
    nc = lib().orc_logup_chunks(ibc, isp, ints, C.c_size_t(air.n_ints), C.c_uint(3), _p(cs))
    assert nc >= 0
    perm = np.empty((4 * (nc + 1), n), dtype=np.uint32)
    cum = np.empty(4, dtype=np.uint32)
    a, b = _u32(alpha_lu), _u32(beta_lu)
    lib().orc_logup_perm_trace(_p(t), C.c_uint(n.bit_length() - 1), ibc, isp, ints, C.c_size_t(air.n_ints), _p(cs),
                               C.c_size_t(nc), _p(a), _p(b), _p(perm), _p(cum))
    return perm, cum, cs[:nc + 1].tolist()


# ---- AVX-512 Montgomery implementations of the heavy primitives (oracle/fast.c): same semantics as the functions above ----
def fast_available():
    lib().orcf_available.restype = C.c_int
    return bool(lib().orcf_available())


def fast_lde_batch(trace, log_blowup=1, shift=GENERATOR):
    t = _u32(trace)
    w, n = t.shape
    out = np.empty((w, n << log_blowup), dtype=np.uint32)
    lib().orcf_lde_batch(_p(t), C.c_uint(n.bit_length() - 1), C.c_size_t(w), C.c_uint(log_blowup), C.c_uint32(shift), _p(out))
    return out


def fast_merkle_commit(mats):
    mats = [_u32(m) for m in mats]
    h = mats[0].shape[1]
    ptrs = (C.c_void_p * len(mats))(*[m.ctypes.data for m in mats])
    widths = (C.c_size_t * len(mats))(*[m.shape[0] for m in mats])
    flat = np.empty((2 * h - 1, 8), dtype=np.uint32)
    lib().orcf_merkle_commit(ptrs, widths, C.c_size_t(len(mats)), C.c_uint(h.bit_length() - 1), _p(flat))
    layers, off, n = [], 0, h
    while n >= 1:
        layers.append(flat[off:off + n])
        off += n
        n >>= 1
    return layers


def fast_constraint_fold(bc, spans, mat, alpha):
    bc, m, al = _u32(bc), _u32(mat), _u32(alpha)
    w, h = m.shape
    out = np.empty((4, h), dtype=np.uint32)
    lib().orcf_constraint_fold(_p(bc), compile_spans(spans), C.c_size_t(len(spans)), _p(m), C.c_size_t(h), _p(al), _p(out))
    return out


def fast_quotient(bc, spans, lde, log_n, alpha, shift=GENERATOR):
    bc, m, al = _u32(bc), _u32(lde), _u32(alpha)
    out = np.empty((2, 4, 1 << log_n), dtype=np.uint32)
    lib().orcf_quotient(_p(bc), compile_spans(spans), C.c_size_t(len(spans)), _p(m), C.c_uint(log_n), C.c_uint(1),
                        C.c_uint32(shift), _p(al), _p(out))
    return out


def fast_eval_at_point(mat, shift, zeta):
    m, z = _u32(mat), _u32(zeta)
    w, n = m.shape
    out = np.empty((w, 4), dtype=np.uint32)
    lib().orcf_eval_at_point(_p(m), C.c_uint(n.bit_length() - 1), C.c_size_t(w), C.c_uint32(shift), _p(z), _p(out))
    return out


def fast_deep_quotient(mats, shift, zeta, gamma, ys):
    mats = [_u32(x) for x in mats]
    m = mats[0].shape[1]
    ptrs = (C.c_void_p * len(mats))(*[x.ctypes.data for x in mats])
    widths = (C.c_size_t * len(mats))(*[x.shape[0] for x in mats])
    z, g, y = _u32(zeta), _u32(gamma), _u32(ys)
    out = np.empty((m, 4), dtype=np.uint32)
    if lib().orcf_deep_quotient(ptrs, widths, C.c_size_t(len(mats)), C.c_uint(m.bit_length() - 1), C.c_uint32(shift), _p(z), _p(g), _p(y), _p(out)):
        raise ValueError("zeta lies on the LDE domain: the reduced opening has no value at one row")
    return out


def big_array(shape):
    """uint32 array backed by orc_big_alloc (2 MB aligned, transparent huge pages advised) -- for the full-size CPU run"""
    n = int(np.prod(shape))
    lib().orc_big_alloc.restype = C.c_void_p
    ptr = lib().orc_big_alloc(C.c_size_t(4 * n))
    buf = (C.c_uint32 * n).from_address(ptr)
    return np.frombuffer(buf, dtype=np.uint32).reshape(shape)


# ---- multi-chip segment under one transcript ----
class ChipC(C.Structure):
    _fields_ = [("air", C.c_void_p), ("trace", C.c_void_p), ("log_n", C.c_uint), ("width", C.c_size_t)]


class ChipsProof(C.Structure):
    _fields_ = [("main_root", C.c_uint32 * 8), ("perm_root", C.c_uint32 * 8), ("quotient_root", C.c_uint32 * 8),
                ("logup_alpha", C.c_uint32 * 4), ("logup_beta", C.c_uint32 * 4), ("alpha", C.c_uint32 * 4), ("zeta", C.c_uint32 * 4), ("gamma", C.c_uint32 * 4),
                ("n_fri_layers", C.c_uint32), ("fri_roots", (C.c_uint32 * 8) * 32), ("fri_betas", (C.c_uint32 * 4) * 32),
                ("final_poly", (C.c_uint32 * 4) * 8), ("final_len", C.c_uint32), ("pow_witness", C.c_uint32),
                ("pow_bits", C.c_uint32), ("n_queries", C.c_uint32), ("n_chips", C.c_uint32), ("log_max", C.c_uint32)]
    VEC = ("main_root", "perm_root", "quotient_root", "logup_alpha", "logup_beta", "alpha", "zeta", "gamma")
    SCALAR = ("n_fri_layers", "final_len", "pow_witness", "pow_bits", "n_queries", "n_chips", "log_max")

    def as_dict(self):
        n = self.n_fri_layers
        d = {k: list(getattr(self, k)) for k in self.VEC}
        d.update({k: int(getattr(self, k)) for k in self.SCALAR})
        d["fri_roots"] = [list(self.fri_roots[i]) for i in range(n)]
        d["fri_betas"] = [list(self.fri_betas[i]) for i in range(n)]
        d["final_poly"] = [list(self.final_poly[i]) for i in range(self.final_len)]
        return d

    @classmethod
    def from_dict(cls, d):
        p = cls()
        for k in cls.VEC:
            for i, v in enumerate(d[k]):
                getattr(p, k)[i] = v
        for k in cls.SCALAR:
            setattr(p, k, d[k])
        for i in range(d["n_fri_layers"]):
            for j in range(8):
                p.fri_roots[i][j] = d["fri_roots"][i][j]
            for j in range(4):
                p.fri_betas[i][j] = d["fri_betas"][i][j]
        for i in range(d["final_len"]):
            for j in range(4):
                p.final_poly[i][j] = d["final_poly"][i][j]
        return p


def _chips_array(chips):
    """chips: list of (trace (W, N), bc, spans, bus) -> (ctypes array, keep-alive list).  bus may already be an Air; for the verifier,
    which reads only the shape, the trace may be given as its shape (W, N)."""
    arr = (ChipC * len(chips))()
    keep = []
    for i, (trace, bc, spans, bus) in enumerate(chips):
        air = bus if isinstance(bus, Air) else Air(bc, spans, bus)
        t = None if isinstance(trace, tuple) else _u32(trace)
        keep.append((air, t))
        w, n = trace if t is None else t.shape
        arr[i].air = C.addressof(air.c)
        arr[i].trace = None if t is None else t.ctypes.data
        arr[i].log_n = n.bit_length() - 1
        arr[i].width = w
    return arr, keep


STAGES = ("lde", "merkle", "logup_gen", "logup_commit", "quotient", "quotient_commit", "openings", "fri_commit", "pow", "query")


def _prove(chips, n_queries, pow_bits, fast, cheat_opening=False):
    """-> (ChipsProof, cumulative sums (K, 4), opened values (n_open, 4), queries (n_queries, words), {stage: seconds})"""
    arr, keep = _chips_array(chips)
    K = len(chips)
    L = lib()
    L.orc_chips_num_opened.restype = C.c_size_t
    L.orc_chips_query_words.restype = C.c_size_t
    n_open = L.orc_chips_num_opened(arr, C.c_size_t(K))
    wpq = L.orc_chips_query_words(arr, C.c_size_t(K))
    proof = ChipsProof()
    cs = np.zeros((K, 4), dtype=np.uint32)
    ys = np.empty((n_open, 4), dtype=np.uint32)
    q = np.empty((n_queries, wpq), dtype=np.uint32)
    st = (C.c_double * 10)()
    prm = ParamsC(n_queries, pow_bits, 1 if fast else 0, 1 if cheat_opening else 0)
    L.orc_prove_chips(arr, C.c_size_t(K), C.byref(prm), C.byref(proof), _p(cs), _p(ys), _p(q), st)
    return proof, cs, ys, q, dict(zip(STAGES, list(st)))


def prove_chips(chips, n_queries=8, pow_bits=4, fast=False):
    """chips: list of (trace, bc, spans, bus) -> (proof dict, cumulative sums (K, 4), opened values (n_open, 4), queries (n_queries, words))"""
    proof, cs, ys, q, _ = _prove(chips, n_queries, pow_bits, fast)
    return proof.as_dict(), cs, ys, q


def verify_chips(chips, proof, cumsums, ys, queries, check_constraints=False):
    """chips: list of (trace-or-shape, bc, spans, bus); only the shape of the trace is used.  0 = accept; see oracle.h for the failure codes"""
    arr, keep = _chips_array(chips)
    p = ChipsProof.from_dict(proof)
    cs, ys, q = _u32(cumsums), _u32(ys), _u32(queries)
    lib().orc_verify_chips.restype = C.c_int
    return lib().orc_verify_chips(arr, C.c_size_t(len(chips)), C.byref(p), _p(cs), _p(ys), _p(q), C.c_int(1 if check_constraints else 0))


# ---- a single segment: the one-chip proof, as the dict the GPU prover returns and the fixtures pin ----
SEGMENT_KEYS = ("trace_root", "logup_alpha", "logup_beta", "perm_root", "cumulative_sum", "alpha", "quotient_root", "zeta", "gamma",
                "n_fri_layers", "final_len", "pow_witness", "pow_bits", "n_queries", "perm_width", "fri_roots", "fri_betas", "final_poly")


def query_words(log_n, width, perm_width=0):
    """words per query of a single segment: r | main row, path | perm row, path (when perm_width) | quotient row, path | FRI layers"""
    log_m = log_n + 1
    return (1 + width + 8 * log_m + (perm_width + 8 * log_m if perm_width else 0) + 8 + 8 * log_m +
            sum(8 + 8 * (log_m - 1 - i) for i in range(log_n)))


def prove(trace, bc, spans, bus=None, n_queries=8, pow_bits=4, fast=False, cheat_opening=False):
    """-> (proof dict, opened values (n_open, 4), query openings (n_queries, words), {stage: seconds})"""
    air = bus if isinstance(bus, Air) else Air(bc, spans, bus)
    proof, cs, ys, q, st = _prove([(trace, bc, spans, air)], n_queries, pow_bits, fast, cheat_opening)
    d = dict(proof.as_dict(), trace_root=list(proof.main_root), cumulative_sum=cs[0].tolist(), perm_width=air.perm_width)
    return {k: d[k] for k in SEGMENT_KEYS}, ys, q, st


def prove_segment(trace, bc, spans, bus=None, n_queries=8, pow_bits=4, fast=False):
    d, _, _, st = prove(trace, bc, spans, bus, n_queries, pow_bits, fast)
    return d, st


def prove_segment_q(trace, bc, spans, n_queries, bus=None, pow_bits=4, fast=False):
    d, ys, q, _ = prove(trace, bc, spans, bus, n_queries, pow_bits, fast)
    return d, ys, q


def verify_segment(bc, spans, log_n, width, proof, ys, queries, check_constraints=False, bus=None):
    """0 = accept; see oracle.h for the failure codes"""
    air = bus if isinstance(bus, Air) else Air(bc, spans, bus)
    if proof["perm_width"] != air.perm_width:
        return 20
    chips_proof = dict(proof, main_root=proof["trace_root"], n_chips=1, log_max=log_n + 1)
    return verify_chips([((width, 1 << log_n), bc, spans, air)], chips_proof, [proof["cumulative_sum"]], ys, queries, check_constraints)
