"""ctypes binding of include/powdr_b200.h -- the Python stand-in for the Rust `extern "C"` block + safe wrappers of
/root/reference/openvm/src/cuda_abi.rs:8-64,97-135,174-223.  Raises if the CUDA library is missing: no CPU fallback."""
import ctypes as C
import os

import numpy as np

P = 2013265921
R_MOD_P = (1 << 32) % P
R_INV_MOD_P = pow(1 << 32, -1, P)
_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_lib", "libpowdr_b200.so")

EXPORTS = [
    "pb_ctx_create", "pb_ctx_destroy", "pb_ctx_synchronize", "pb_ctx_set_poseidon2", "pb_host_alloc", "pb_host_free",
    "pb_device_alloc", "pb_device_free", "pb_copy_h2d", "pb_copy_d2h", "pb_memset_zero", "pb_to_monty", "pb_from_monty",
    "pb_lde_batch", "pb_air_compile", "pb_air_free", "pb_air_is_jit", "pb_air_jit_compile_only", "pb_quotient", "pb_constraint_fold", "pb_merkle_commit",
    "pb_merkle_commit_rows8", "pb_poseidon2_permute", "pb_fri_fold", "pb_eval_at_point", "pb_deep_quotient", "pb_prove_segment", "pb_query_words", "pb_query_segment", "pb_last_openings", "pb_last_stage_ms",
    "pb_ctx_set_fri_params", "pb_air_set_interactions", "pb_air_perm_width", "pb_air_logup_compile_only", "pb_allgather_caps", "pb_bus_compile", "pb_bus_free", "pb_bus_apply",
    "pb_shard_columns", "pb_lde_shard", "pb_prove_segment_sharded", "pb_query_segment_sharded", "pb_prove_chips", "pb_prove_chips_host", "pb_chips_sizes", "pb_query_chips", "pb_host_poseidon2_permute",
    "pb_prove_chips_sharded", "pb_query_chips_sharded", "pb_ctx_set_memory_budget", "pb_last_row_blocks", "pb_footprint_bytes",
    "pb_footprint_bytes_sharded",
    "pb_launch_count", "pb_leaf_kernel_profile", "_apc_tracegen", "_apc_apply_derived_expr", "_apc_apply_bus",
    "pb_vk_create", "pb_vk_free", "pb_verify_chips", "pb_verify_segment",
    "pb_chips_proof_encode", "pb_segment_proof_encode", "pb_proof_bytes_sizes", "pb_chips_proof_decode", "pb_segment_proof_decode",
    "pb_verify_proof_bytes",
    "pb_group_create", "pb_group_destroy", "pb_prove_chips_group", "pb_query_chips_group",
]
PB_ERR_INVALID_ARG = -1
PB_ERR_UNSUPPORTED = -2
PB_ERR_COMM = -6
PB_ERR_INTERNAL = -7
PB_ERR_REJECTED = -8
PB_PROOF_MAGIC = 0x46504250
PB_PROOF_VERSION = 1
PB_PROOF_MAX_CHIPS = 4096
REASON_MALFORMED = 23


class LibraryMissing(RuntimeError):
    pass


class PbError(RuntimeError):
    def __init__(self, code, where):
        super().__init__("%s failed with code %d (%s)" % (where, code, "cudaError_t" if code > 0 else "PB_ERR"))
        self.code = code


class ProofRejected(PbError):
    """PB_ERR_REJECTED from a decoder: .reason is 23 for malformed bytes, 20 for a blob of another shape"""

    def __init__(self, reason, where):
        super().__init__(PB_ERR_REJECTED, "%s (reason %d)" % (where, reason))
        self.reason = reason


class Span(C.Structure):
    _fields_ = [("off", C.c_uint32), ("len", C.c_uint32)]


class OriginalAir(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("buffer", C.c_void_p), ("row_block_size", C.c_int)]


class Subst(C.Structure):
    _fields_ = [("air_index", C.c_int), ("col", C.c_int), ("row", C.c_int), ("apc_col", C.c_int)]


class DerivedExprSpec(C.Structure):
    _fields_ = [("col_base", C.c_uint64), ("span", Span)]


class DevInteraction(C.Structure):
    _fields_ = [("bus_id", C.c_uint32), ("num_args", C.c_uint32), ("args_index_off", C.c_uint32)]


class SegmentProof(C.Structure):
    """pb_segment_proof_t (include/powdr_b200.h)"""
    _fields_ = [("trace_root", C.c_uint32 * 8), ("logup_alpha", C.c_uint32 * 4), ("logup_beta", C.c_uint32 * 4),
                ("perm_root", C.c_uint32 * 8), ("cumulative_sum", C.c_uint32 * 4), ("alpha", C.c_uint32 * 4),
                ("quotient_root", C.c_uint32 * 8), ("zeta", C.c_uint32 * 4), ("gamma", C.c_uint32 * 4),
                ("n_fri_layers", C.c_uint32), ("fri_roots", (C.c_uint32 * 8) * 32), ("fri_betas", (C.c_uint32 * 4) * 32),
                ("final_poly", (C.c_uint32 * 4) * 8), ("final_len", C.c_uint32), ("pow_witness", C.c_uint32),
                ("pow_bits", C.c_uint32), ("n_queries", C.c_uint32), ("perm_width", C.c_uint32)]
    VEC = ("trace_root", "logup_alpha", "logup_beta", "perm_root", "cumulative_sum", "alpha", "quotient_root", "zeta", "gamma")
    SCALAR = ("n_fri_layers", "final_len", "pow_witness", "pow_bits", "n_queries", "perm_width")

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
        """the struct of an as_dict() result"""
        p = cls()
        for k in cls.VEC:
            getattr(p, k)[:] = [int(v) for v in d[k]]
        for k in cls.SCALAR:
            setattr(p, k, int(d[k]))
        for name, rows in (("fri_roots", d["fri_roots"]), ("fri_betas", d["fri_betas"]), ("final_poly", d["final_poly"])):
            for i, row in enumerate(rows):
                getattr(p, name)[i][:] = [int(v) for v in row]
        return p


class Chip(C.Structure):
    """pb_chip_t"""
    _fields_ = [("air", C.c_void_p), ("d_trace", C.c_void_p), ("log_n", C.c_size_t), ("width", C.c_size_t)]


class ChipsProof(C.Structure):
    """pb_chips_proof_t (include/powdr_b200.h)"""
    _fields_ = [("main_root", C.c_uint32 * 8), ("perm_root", C.c_uint32 * 8), ("quotient_root", C.c_uint32 * 8),
                ("logup_alpha", C.c_uint32 * 4), ("logup_beta", C.c_uint32 * 4), ("alpha", C.c_uint32 * 4), ("zeta", C.c_uint32 * 4),
                ("gamma", C.c_uint32 * 4), ("n_fri_layers", C.c_uint32), ("fri_roots", (C.c_uint32 * 8) * 32),
                ("fri_betas", (C.c_uint32 * 4) * 32), ("final_poly", (C.c_uint32 * 4) * 8), ("final_len", C.c_uint32),
                ("pow_witness", C.c_uint32), ("pow_bits", C.c_uint32), ("n_queries", C.c_uint32), ("n_chips", C.c_uint32), ("log_max", C.c_uint32)]
    VEC = ("main_root", "perm_root", "quotient_root", "logup_alpha", "logup_beta", "alpha", "zeta", "gamma")
    SCALAR = ("n_fri_layers", "final_len", "pow_witness", "pow_bits", "n_queries", "n_chips", "log_max")
    as_dict = SegmentProof.as_dict
    from_dict = classmethod(SegmentProof.from_dict.__func__)


class VerifyChip(C.Structure):
    """pb_verify_chip_t"""
    _fields_ = [("vk", C.c_void_p), ("log_n", C.c_size_t)]


class VerifyParams(C.Structure):
    """pb_verify_params_t"""
    _fields_ = [("n_queries", C.c_uint32), ("pow_bits", C.c_uint32), ("rc_ext", C.c_void_p), ("rc_int", C.c_void_p), ("diag_m1", C.c_void_p)]


class ProofChip(C.Structure):
    """pb_proof_chip_t: a chip's shape as the proof's byte form carries it"""
    _fields_ = [("log_n", C.c_uint32), ("width", C.c_uint32), ("perm_width", C.c_uint32)]


STAGES = ("h2d", "lde", "merkle", "logup_gen", "logup_commit", "quotient", "qlde", "qmerkle", "open", "fri", "pow", "total")


_lib = None


def footprint_bytes(chips, log_blocks=0):
    """chips: [(log_n, width, perm_width)] -> the device bytes pb_footprint_bytes counts for a proof of them in 2^log_blocks row blocks"""
    lib = load_library()
    k = len(chips)
    ln, w, wp = [(C.c_size_t * k)(*[int(c[i]) for c in chips]) for i in range(3)]
    out = C.c_size_t()
    _chk(lib.pb_footprint_bytes(ln, w, wp, C.c_size_t(k), C.c_uint32(log_blocks), C.byref(out)), "pb_footprint_bytes")
    return int(out.value)


def footprint_bytes_sharded(chips, world, log_blocks=0):
    """chips: [(log_n, width, perm_width)] -> one rank's device bytes pb_footprint_bytes_sharded counts for a proof of them on `world`
    ranks with each rank block in 2^log_blocks sub-blocks (the caller's column share not included)"""
    lib = load_library()
    k = len(chips)
    ln, w, wp = [(C.c_size_t * k)(*[int(c[i]) for c in chips]) for i in range(3)]
    out = C.c_size_t()
    _chk(lib.pb_footprint_bytes_sharded(ln, w, wp, C.c_size_t(k), C.c_int(world), C.c_uint32(log_blocks), C.byref(out)),
         "pb_footprint_bytes_sharded")
    return int(out.value)


def load_library(path=None):
    """dlopen the in-tree sm_90a library; never falls back to anything else."""
    global _lib
    if _lib is not None:
        return _lib
    path = path or LIB_PATH
    if not os.path.exists(path):
        raise LibraryMissing("%s not built: run `python -m powdr_b200.build` (nvcc, sm_90a)" % path)
    lib = C.CDLL(path)
    for name in EXPORTS:
        if not hasattr(lib, name):
            raise LibraryMissing("symbol %s missing from %s" % (name, path))
        getattr(lib, name).restype = C.c_int
    lib.pb_launch_count.restype = C.c_uint64
    _lib = lib
    return lib


def _chk(code, where):
    if code != 0:
        raise PbError(code, where)


def _u32(a):
    return np.ascontiguousarray(a, dtype=np.uint32)


class DeviceBuffer:
    """Caller-owned device memory (DeviceBuffer<T> of openvm-cuda-common)."""

    def __init__(self, ctx, nbytes):
        self.ctx, self.nbytes = ctx, int(nbytes)
        p = C.c_void_p()
        _chk(ctx.lib.pb_device_alloc(C.byref(p), C.c_size_t(max(4, self.nbytes))), "pb_device_alloc")
        self.ptr = p.value

    def free(self):
        if self.ptr:
            self.ctx.lib.pb_device_free(C.c_void_p(self.ptr))
            self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass

    def upload(self, arr):
        a = np.ascontiguousarray(arr)
        assert a.nbytes <= self.nbytes
        _chk(self.ctx.lib.pb_copy_h2d(self.ctx.h, C.c_void_p(self.ptr), a.ctypes.data_as(C.c_void_p), C.c_size_t(a.nbytes)), "pb_copy_h2d")
        self.ctx.synchronize()
        return self

    def download(self, shape, dtype=np.uint32):
        out = np.empty(shape, dtype=dtype)
        assert out.nbytes <= self.nbytes
        _chk(self.ctx.lib.pb_copy_d2h(self.ctx.h, out.ctypes.data_as(C.c_void_p), C.c_void_p(self.ptr), C.c_size_t(out.nbytes)), "pb_copy_d2h")
        return out

    def zero(self):
        _chk(self.ctx.lib.pb_memset_zero(self.ctx.h, C.c_void_p(self.ptr), C.c_size_t(self.nbytes)), "pb_memset_zero")
        return self


class Air:
    def __init__(self, ctx, bytecode, spans, width, bus=None):
        """bus: (interactions [(bus_id, num_args, args_index_off)], arg_spans [(off, len)], bytecode) as returned by
        powdr_b200.machine.compile_bus(machine, 1) -- attaches the AIR's bus interactions (LogUp phase of the prover)"""
        self.ctx, self.width, self.n_constraints = ctx, width, len(spans)
        bc = _u32(bytecode)
        sp = (Span * max(1, len(spans)))()
        for i, (o, l) in enumerate(spans):
            sp[i].off, sp[i].len = o, l
        h = C.c_void_p()
        _chk(ctx.lib.pb_air_compile(ctx.h, bc.ctypes.data_as(C.c_void_p), C.c_size_t(bc.size), sp, C.c_size_t(len(spans)),
                                    C.c_uint32(width), C.byref(h)), "pb_air_compile")
        self.h = h
        self.perm_width = 0
        if bus and len(bus[0]):
            ints, isp, ibc = bus
            ibc = _u32(ibc)
            spn = (Span * max(1, len(isp)))()
            for i, (o, l) in enumerate(isp):
                spn[i].off, spn[i].len = o, l
            di = (DevInteraction * len(ints))()
            for i, (b, n, o) in enumerate(ints):
                di[i].bus_id, di[i].num_args, di[i].args_index_off = b, n, o
            _chk(ctx.lib.pb_air_set_interactions(ctx.h, self.h, ibc.ctypes.data_as(C.c_void_p), C.c_size_t(ibc.size), spn, C.c_size_t(len(isp)),
                                                 di, C.c_size_t(len(ints))), "pb_air_set_interactions")
            wp = C.c_size_t()
            _chk(ctx.lib.pb_air_perm_width(self.h, C.byref(wp)), "pb_air_perm_width")
            self.perm_width = int(wp.value)

    @property
    def is_jit(self):
        return bool(self.ctx.lib.pb_air_is_jit(self.h))

    def free(self):
        if self.h:
            self.ctx.lib.pb_air_free(self.h)
            self.h = None


class VerifyingKey:
    """pb_vk_t: what the host verifier reads of an AIR, from the same (bytecode, spans, width, bus) as Context.air.  Needs no GPU."""

    def __init__(self, bytecode, spans, width, bus=None):
        self.lib = load_library()
        bc = _u32(bytecode)
        sp = (Span * max(1, len(spans)))(*[Span(o, l) for o, l in spans])
        ints, isp, ibc = bus if bus and len(bus[0]) else ([], [], [])
        ibc = _u32(ibc)
        spn = (Span * max(1, len(isp)))(*[Span(o, l) for o, l in isp])
        di = (DevInteraction * max(1, len(ints)))(*[DevInteraction(b, n, o) for b, n, o in ints])
        h = C.c_void_p()
        _chk(self.lib.pb_vk_create(bc.ctypes.data_as(C.c_void_p), C.c_size_t(bc.size), sp, C.c_size_t(len(spans)), C.c_uint32(width),
                                   ibc.ctypes.data_as(C.c_void_p), C.c_size_t(ibc.size), spn, C.c_size_t(len(isp)), di, C.c_size_t(len(ints)),
                                   C.byref(h)), "pb_vk_create")
        self.h = h

    def free(self):
        if self.h:
            self.lib.pb_vk_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def _verify_params(n_queries, pow_bits, poseidon2):
    """-> (pb_verify_params_t, keep-alive); poseidon2 = (rc_ext [8][16], rc_int [13], diag_m1 [16]) canonical, or None for the default"""
    prm = VerifyParams(n_queries, pow_bits, None, None, None)
    keep = [_u32(a) for a in poseidon2] if poseidon2 is not None else []
    if keep:
        assert keep[0].size == 128 and keep[1].size == 13 and keep[2].size == 16
        prm.rc_ext, prm.rc_int, prm.diag_m1 = [a.ctypes.data for a in keep]
    return prm, keep


def verify_chips(chips, proof, cumsums, ys, queries, n_queries=100, pow_bits=16, poseidon2=None):
    """pb_verify_chips on the host: chips [(VerifyingKey, log_n)]; proof, cumulative sums, opened values and queries as
    Context.prove_chips returns them; n_queries / pow_bits: the security parameters the proof must have.
    -> (rc, reason): (0, 0) accepted, (PB_ERR_REJECTED, the failed check), or (PB_ERR_INVALID_ARG, 0)"""
    lib = load_library()
    arr = (VerifyChip * max(1, len(chips)))(*[VerifyChip(vk.h.value, int(ln)) for vk, ln in chips])
    p = proof if isinstance(proof, ChipsProof) else ChipsProof.from_dict(proof)
    prm, keep = _verify_params(n_queries, pow_bits, poseidon2)
    cs, y, q = _u32(cumsums), _u32(ys), _u32(queries)
    reason = C.c_int()
    rc = lib.pb_verify_chips(arr, C.c_size_t(len(chips)), C.byref(prm), C.byref(p), cs.ctypes.data_as(C.c_void_p), y.ctypes.data_as(C.c_void_p),
                             C.c_size_t(y.size), q.ctypes.data_as(C.c_void_p), C.c_size_t(q.size), C.byref(reason))
    return rc, reason.value


def verify_segment(vk, log_n, proof, ys, queries, n_queries=100, pow_bits=16, poseidon2=None):
    """pb_verify_segment: a proof, opened values and queries as Context.prove_segment / query_segment return them -> (rc, reason)"""
    lib = load_library()
    p = proof if isinstance(proof, SegmentProof) else SegmentProof.from_dict(proof)
    prm, keep = _verify_params(n_queries, pow_bits, poseidon2)
    y, q = _u32(ys), _u32(queries)
    reason = C.c_int()
    rc = lib.pb_verify_segment(vk.h, C.c_size_t(log_n), C.byref(prm), C.byref(p), y.ctypes.data_as(C.c_void_p), C.c_size_t(y.size),
                               q.ctypes.data_as(C.c_void_p), C.c_size_t(q.size), C.byref(reason))
    return rc, reason.value


# ---- the proof's byte form (include/powdr_b200.h) ----
def _encode(call, where):
    """call(out, capacity, len_ptr) twice: the size, then the bytes"""
    n = C.c_size_t()
    _chk(call(None, C.c_size_t(0), C.byref(n)), where)
    out = C.create_string_buffer(n.value)
    _chk(call(out, C.c_size_t(n.value), C.byref(n)), where)
    return out.raw[:n.value]


def encode_chips_proof(proof, chips, cumsums, ys, queries):
    """pb_chips_proof_encode: proof, cumulative sums, opened values and queries as Context.prove_chips returns them; chips
    [(log_n, width, perm_width)] -> bytes"""
    lib = load_library()
    p = proof if isinstance(proof, ChipsProof) else ChipsProof.from_dict(proof)
    arr = (ProofChip * max(1, len(chips)))(*[ProofChip(*[int(v) for v in c]) for c in chips])
    cs, y, q = _u32(cumsums), _u32(ys), _u32(queries if queries is not None else np.empty(0))
    return _encode(lambda out, cap, n: lib.pb_chips_proof_encode(
        C.byref(p), arr, C.c_size_t(len(chips)), cs.ctypes.data_as(C.c_void_p), y.ctypes.data_as(C.c_void_p), C.c_size_t(y.size),
        q.ctypes.data_as(C.c_void_p), C.c_size_t(q.size), out, cap, n), "pb_chips_proof_encode")


def encode_segment_proof(proof, log_n, width, ys, queries):
    """pb_segment_proof_encode: a proof, opened values and queries as Context.prove_segment / query_segment return them -> bytes"""
    lib = load_library()
    p = proof if isinstance(proof, SegmentProof) else SegmentProof.from_dict(proof)
    y, q = _u32(ys), _u32(queries)
    return _encode(lambda out, cap, n: lib.pb_segment_proof_encode(
        C.byref(p), C.c_size_t(log_n), C.c_size_t(width), y.ctypes.data_as(C.c_void_p), C.c_size_t(y.size), q.ctypes.data_as(C.c_void_p),
        C.c_size_t(q.size), out, cap, n), "pb_segment_proof_encode")


def decode_proof(blob, segment=False):
    """pb_proof_bytes_sizes + pb_chips_proof_decode -> (proof dict, chips [(log_n, width, perm_width)], cumulative sums (K, 4),
    opened values (n_opened, 4), queries (n_queries, words_per_query)); segment=True: pb_segment_proof_decode -> (segment proof dict,
    log_n, width, opened values, queries).  Raises ProofRejected for bytes the decoder refuses."""
    lib = load_library()
    b = bytes(blob)
    k, nys, nq, reason = C.c_size_t(), C.c_size_t(), C.c_size_t(), C.c_int()
    rc = lib.pb_proof_bytes_sizes(b, C.c_size_t(len(b)), C.byref(k), C.byref(nys), C.byref(nq), C.byref(reason))
    if rc == PB_ERR_REJECTED:
        raise ProofRejected(reason.value, "pb_proof_bytes_sizes")
    _chk(rc, "pb_proof_bytes_sizes")
    n_q = int.from_bytes(b[12:16], "little")          # header word 3, of a blob the call above has checked
    ys = np.empty((nys.value // 4, 4), dtype=np.uint32)
    q = np.empty((n_q, nq.value // n_q if n_q else 0), dtype=np.uint32)
    yp, qp = ys.ctypes.data_as(C.c_void_p), q.ctypes.data_as(C.c_void_p)
    if segment:
        proof, log_n, width = SegmentProof(), C.c_size_t(), C.c_size_t()
        rc = lib.pb_segment_proof_decode(b, C.c_size_t(len(b)), C.byref(proof), C.byref(log_n), C.byref(width), yp, nys, qp, nq, C.byref(reason))
        out = (proof, int(log_n.value), int(width.value), ys, q)
    else:
        proof, chips, cs = ChipsProof(), (ProofChip * k.value)(), np.empty((k.value, 4), dtype=np.uint32)
        rc = lib.pb_chips_proof_decode(b, C.c_size_t(len(b)), C.byref(proof), chips, k, cs.ctypes.data_as(C.c_void_p), yp, nys, qp, nq,
                                       C.byref(reason))
        out = (proof, [(c.log_n, c.width, c.perm_width) for c in chips], cs, ys, q)
    if rc == PB_ERR_REJECTED:
        raise ProofRejected(reason.value, "pb_segment_proof_decode" if segment else "pb_chips_proof_decode")
    _chk(rc, "pb_segment_proof_decode" if segment else "pb_chips_proof_decode")
    return (out[0].as_dict(),) + out[1:]


def verify_proof_bytes(vks, blob, n_queries=100, pow_bits=16, poseidon2=None):
    """pb_verify_proof_bytes: vks [VerifyingKey], one per chip of the blob in its order -> (rc, reason) as verify_chips"""
    lib = load_library()
    arr = (C.c_void_p * max(1, len(vks)))(*[vk.h.value for vk in vks])
    prm, keep = _verify_params(n_queries, pow_bits, poseidon2)
    b = bytes(blob)
    reason = C.c_int()
    rc = lib.pb_verify_proof_bytes(arr, C.c_size_t(len(vks)), C.byref(prm), b, C.c_size_t(len(b)), C.byref(reason))
    return rc, reason.value


class Context:
    """pb_ctx_t: one per GPU / stream."""

    def __init__(self, device=0, stream=None):
        self.lib = load_library()
        h = C.c_void_p()
        _chk(self.lib.pb_ctx_create(C.byref(h), C.c_int(device), C.c_void_p(stream or 0)), "pb_ctx_create")
        self.h = h
        self.device = device
        self.n_queries = 100

    def close(self):
        if self.h:
            self.lib.pb_ctx_destroy(self.h)
            self.h = None

    def synchronize(self):
        _chk(self.lib.pb_ctx_synchronize(self.h), "pb_ctx_synchronize")

    # ---- memory ----
    def alloc(self, nbytes):
        return DeviceBuffer(self, nbytes)

    def to_device(self, arr, monty=True):
        """numpy (canonical) -> device buffer (Montgomery unless monty=False); conversion done on the host."""
        a = _u32(arr)
        if monty:
            a = ((a.astype(np.uint64) * np.uint64(R_MOD_P)) % np.uint64(P)).astype(np.uint32)
        return DeviceBuffer(self, a.nbytes).upload(a)

    def to_host(self, buf, shape, monty=True):
        raw = buf.download(shape)
        if monty:
            raw = ((raw.astype(np.uint64) * np.uint64(R_INV_MOD_P)) % np.uint64(P)).astype(np.uint32)
        return raw

    # ---- stages ----
    def air(self, bytecode, spans, width, bus=None):
        return Air(self, bytecode, spans, width, bus)

    def set_fri_params(self, n_queries, pow_bits):
        _chk(self.lib.pb_ctx_set_fri_params(self.h, C.c_uint32(n_queries), C.c_uint32(pow_bits)), "pb_ctx_set_fri_params")
        self.n_queries = n_queries

    def lde_batch(self, d_trace_ptr, log_n, width, d_lde_ptr, log_blowup=1, shift=31):
        _chk(self.lib.pb_lde_batch(self.h, C.c_void_p(d_trace_ptr), C.c_size_t(log_n), C.c_size_t(width), C.c_uint32(log_blowup),
                                   C.c_uint32(shift), C.c_void_p(d_lde_ptr)), "pb_lde_batch")

    def quotient(self, air, d_lde_ptr, log_n, alpha, d_q_ptr, log_blowup=1, shift=31):
        al = (C.c_uint32 * 4)(*[int(x) for x in alpha])
        _chk(self.lib.pb_quotient(self.h, air.h, C.c_void_p(d_lde_ptr), C.c_size_t(log_n), C.c_uint32(log_blowup), C.c_uint32(shift),
                                  al, C.c_void_p(d_q_ptr)), "pb_quotient")

    def constraint_fold(self, air, d_mat_ptr, height, alpha, d_out_ptr):
        al = (C.c_uint32 * 4)(*[int(x) for x in alpha])
        _chk(self.lib.pb_constraint_fold(self.h, air.h, C.c_void_p(d_mat_ptr), C.c_size_t(height), al, C.c_void_p(d_out_ptr)),
             "pb_constraint_fold")

    def merkle_commit(self, mat_ptrs, widths, log_h, d_layers_ptr, want_root=True):
        n = len(mat_ptrs)
        ptrs = (C.c_void_p * n)(*mat_ptrs)
        ws = (C.c_size_t * n)(*widths)
        root = (C.c_uint32 * 8)()
        _chk(self.lib.pb_merkle_commit(self.h, ptrs, ws, C.c_size_t(n), C.c_size_t(log_h), C.c_void_p(d_layers_ptr),
                                       root if want_root else None), "pb_merkle_commit")
        return list(root) if want_root else None

    def merkle_commit_rows8(self, d_rows_ptr, log_h, d_layers_ptr, want_root=True):
        root = (C.c_uint32 * 8)()
        _chk(self.lib.pb_merkle_commit_rows8(self.h, C.c_void_p(d_rows_ptr), C.c_size_t(log_h), C.c_void_p(d_layers_ptr),
                                             root if want_root else None), "pb_merkle_commit_rows8")
        return list(root) if want_root else None

    def poseidon2_permute(self, d_states_ptr, n, reps=1):
        _chk(self.lib.pb_poseidon2_permute(self.h, C.c_void_p(d_states_ptr), C.c_size_t(n), C.c_int(reps)), "pb_poseidon2_permute")

    def fri_fold(self, d_in_ptr, log_len, shift, beta, d_out_ptr):
        b = (C.c_uint32 * 4)(*[int(x) for x in beta])
        _chk(self.lib.pb_fri_fold(self.h, C.c_void_p(d_in_ptr), C.c_size_t(log_len), C.c_uint32(shift), b, C.c_void_p(d_out_ptr)),
             "pb_fri_fold")

    def eval_at_point(self, d_mat_ptr, log_n, width, shift, zeta, d_ys_ptr):
        z = (C.c_uint32 * 4)(*[int(x) for x in zeta])
        _chk(self.lib.pb_eval_at_point(self.h, C.c_void_p(d_mat_ptr), C.c_size_t(log_n), C.c_size_t(width), C.c_uint32(shift), z,
                                       C.c_void_p(d_ys_ptr)), "pb_eval_at_point")

    def deep_quotient(self, mat_ptrs, widths, log_m, shift, zeta, gamma, d_ys_ptr, d_out_ptr):
        n = len(mat_ptrs)
        ptrs = (C.c_void_p * n)(*mat_ptrs)
        ws = (C.c_size_t * n)(*widths)
        z = (C.c_uint32 * 4)(*[int(x) for x in zeta])
        g = (C.c_uint32 * 4)(*[int(x) for x in gamma])
        _chk(self.lib.pb_deep_quotient(self.h, ptrs, ws, C.c_size_t(n), C.c_size_t(log_m), C.c_uint32(shift), z, g, C.c_void_p(d_ys_ptr),
                                       C.c_void_p(d_out_ptr)), "pb_deep_quotient")

    def prove_segment(self, air, trace_ptr, log_n, width, on_device=False):
        proof = SegmentProof()
        _chk(self.lib.pb_prove_segment(self.h, air.h, C.c_void_p(trace_ptr), C.c_size_t(log_n), C.c_size_t(width),
                                       C.c_uint32(1 if on_device else 0), C.byref(proof)), "pb_prove_segment")
        return proof.as_dict()

    def lde_shard(self, d_trace_ptr, log_n, width, world, blk, d_out_ptr, shift=31):
        _chk(self.lib.pb_lde_shard(self.h, C.c_void_p(d_trace_ptr), C.c_size_t(log_n), C.c_size_t(width), C.c_uint32(shift), C.c_int(world),
                                   C.c_int(blk), C.c_void_p(d_out_ptr)), "pb_lde_shard")

    def prove_segment_sharded(self, air, trace_cols_ptr, log_n, width, comm, on_device=False):
        """one rank of a multi-GPU segment proof; comm: powdr_b200.sharded.Comm.  trace_cols_ptr: this rank's column block."""
        proof = SegmentProof()
        _chk(self.lib.pb_prove_segment_sharded(self.h, air.h, C.c_void_p(trace_cols_ptr or 0), C.c_size_t(log_n), C.c_size_t(width),
                                               C.c_uint32(1 if on_device else 0), C.byref(comm.c), C.byref(proof)), "pb_prove_segment_sharded")
        return proof.as_dict()

    def query_segment_sharded(self, comm, log_n, width, perm_width=0):
        """query openings of the last prove_segment_sharded (collective: every rank calls it, every rank gets the whole set)"""
        wpq = C.c_size_t()
        _chk(self.lib.pb_query_words(C.c_size_t(log_n), C.c_size_t(width), C.c_size_t(perm_width), C.byref(wpq)), "pb_query_words")
        out = np.empty((self.n_queries, wpq.value), dtype=np.uint32)
        _chk(self.lib.pb_query_segment_sharded(self.h, C.byref(comm.c), out.ctypes.data_as(C.c_void_p), C.c_size_t(out.size)), "pb_query_segment_sharded")
        return out

    def query_segment(self, log_n, width, perm_width=0):
        """-> (n_queries, words_per_query) uint32 array of openings for the last prove_segment (n_queries from set_fri_params),
        and the opened values (width + 2*perm_width + 8, 4)"""
        wpq = C.c_size_t()
        _chk(self.lib.pb_query_words(C.c_size_t(log_n), C.c_size_t(width), C.c_size_t(perm_width), C.byref(wpq)), "pb_query_words")
        out = np.empty((self.n_queries, wpq.value), dtype=np.uint32)
        _chk(self.lib.pb_query_segment(self.h, out.ctypes.data_as(C.c_void_p), C.c_size_t(out.size)), "pb_query_segment")
        ys = np.empty((width + 2 * perm_width + 8, 4), dtype=np.uint32)
        _chk(self.lib.pb_last_openings(self.h, ys.ctypes.data_as(C.c_void_p), C.c_size_t(ys.size)), "pb_last_openings")
        return out, ys

    def prove_chips(self, chips, want_queries=True, on_device=True):
        """chips: [(Air, trace_ptr, log_n, width)], Montgomery traces, device-resident (pb_prove_chips) or, on_device=False, in host
        memory (pb_prove_chips_host: the same proof, copied in behind the work; pinned memory overlaps the copy).  All chips of a segment
        under one transcript.  -> (proof dict, cumulative sums (K, 4), opened values (n_opened, 4), queries (n_queries, words) or None)"""
        K = len(chips)
        arr = (Chip * K)(*[Chip(a.h.value, int(p), int(ln), int(w)) for a, p, ln, w in chips])
        proof = ChipsProof()
        cums = np.zeros((K, 4), dtype=np.uint32)
        name = "pb_prove_chips" if on_device else "pb_prove_chips_host"
        _chk(getattr(self.lib, name)(self.h, arr, C.c_size_t(K), C.byref(proof), cums.ctypes.data_as(C.c_void_p)), name)
        n_open, wpq = C.c_size_t(), C.c_size_t()
        _chk(self.lib.pb_chips_sizes(arr, C.c_size_t(K), C.byref(n_open), C.byref(wpq)), "pb_chips_sizes")
        ys = np.empty((n_open.value, 4), dtype=np.uint32)
        q = np.empty((self.n_queries, wpq.value), dtype=np.uint32) if want_queries and self.n_queries else None
        _chk(self.lib.pb_query_chips(self.h, q.ctypes.data_as(C.c_void_p) if q is not None else None, C.c_size_t(q.size if q is not None else 0),
                                     ys.ctypes.data_as(C.c_void_p), C.c_size_t(ys.size)), "pb_query_chips")
        return proof.as_dict(), cums, ys, q

    def prove_chips_sharded(self, chips, comm, want_queries=True):
        """one rank of a multi-GPU proof of all chips under one transcript (pb_prove_chips_sharded); comm: powdr_b200.sharded.Comm.
        chips: [(Air, d_trace_ptr, log_n, width)] in the same order on every rank, d_trace_ptr = this rank's column block of the chip
        (device, Montgomery; 0 when empty), width = the whole width.  -> the tuple of prove_chips, equal to it on every rank"""
        K = len(chips)
        arr = (Chip * K)(*[Chip(a.h.value, int(p or 0), int(ln), int(w)) for a, p, ln, w in chips])
        proof = ChipsProof()
        cums = np.zeros((K, 4), dtype=np.uint32)
        _chk(self.lib.pb_prove_chips_sharded(self.h, arr, C.c_size_t(K), C.byref(comm.c), C.byref(proof), cums.ctypes.data_as(C.c_void_p)),
             "pb_prove_chips_sharded")
        ys, q = self.query_chips_sharded(comm, arr, want_queries)
        return proof.as_dict(), cums, ys, q

    def query_chips_sharded(self, comm, chip_arr, want_queries=True):
        """opened values and query openings of the last prove_chips_sharded (collective when queries are asked for)"""
        n_open, wpq = C.c_size_t(), C.c_size_t()
        _chk(self.lib.pb_chips_sizes(chip_arr, C.c_size_t(len(chip_arr)), C.byref(n_open), C.byref(wpq)), "pb_chips_sizes")
        ys = np.empty((n_open.value, 4), dtype=np.uint32)
        q = np.empty((self.n_queries, wpq.value), dtype=np.uint32) if want_queries and self.n_queries else None
        _chk(self.lib.pb_query_chips_sharded(self.h, C.byref(comm.c), q.ctypes.data_as(C.c_void_p) if q is not None else None,
                                             C.c_size_t(q.size if q is not None else 0), ys.ctypes.data_as(C.c_void_p), C.c_size_t(ys.size)),
             "pb_query_chips_sharded")
        return ys, q

    def set_memory_budget(self, nbytes):
        """device memory the single-GPU provers may use (0: free memory at the call + what the context holds); nonzero also governs
        the sharded provers, per rank, and must then be the same on every rank (0: they stay resident)"""
        _chk(self.lib.pb_ctx_set_memory_budget(self.h, C.c_size_t(int(nbytes))), "pb_ctx_set_memory_budget")

    def last_row_blocks(self):
        """log2 of the row blocks of the last prove_segment / prove_chips, or of the sub-blocks per rank of a sharded proof (0: resident)"""
        lb = C.c_uint32()
        _chk(self.lib.pb_last_row_blocks(self.h, C.byref(lb)), "pb_last_row_blocks")
        return int(lb.value)

    def last_stage_ms(self):
        ms = (C.c_float * len(STAGES))()
        _chk(self.lib.pb_last_stage_ms(self.h, ms), "pb_last_stage_ms")
        return dict(zip(STAGES, [float(x) for x in ms]))

    def launch_count(self):
        return int(self.lib.pb_launch_count(self.h))

    def leaf_kernel_profile(self):
        n, ms, by = C.c_int(), C.c_double(), C.c_double()
        _chk(self.lib.pb_leaf_kernel_profile(self.h, C.byref(n), C.byref(ms), C.byref(by)), "pb_leaf_kernel_profile")
        return n.value, ms.value, by.value

    def host_alloc(self, nbytes):
        p = C.c_void_p()
        _chk(self.lib.pb_host_alloc(C.byref(p), C.c_size_t(nbytes)), "pb_host_alloc")
        return p.value

    def host_free(self, ptr):
        self.lib.pb_host_free(C.c_void_p(ptr))

    # ---- stage 0, generated periphery kernel ----
    def bus_compile(self, bus, width, var_bus=3, tuple2_bus=7, bitwise_bus=6):
        """bus = machine.compile_bus(machine, 1) -> opaque handle for bus_apply"""
        ints, isp, ibc = bus
        ibc = _u32(ibc)
        spn = (Span * max(1, len(isp)))()
        for i, (o, l) in enumerate(isp):
            spn[i].off, spn[i].len = o, l
        di = (DevInteraction * max(1, len(ints)))()
        for i, (b, n, o) in enumerate(ints):
            di[i].bus_id, di[i].num_args, di[i].args_index_off = b, n, o
        h = C.c_void_p()
        _chk(self.lib.pb_bus_compile(self.h, ibc.ctypes.data_as(C.c_void_p), C.c_size_t(ibc.size), spn, C.c_size_t(len(isp)), di, C.c_size_t(len(ints)),
                                     C.c_uint32(width), C.c_uint32(var_bus), C.c_uint32(tuple2_bus), C.c_uint32(bitwise_bus), C.byref(h)), "pb_bus_compile")
        return h

    def bus_apply(self, handle, d_trace_ptr, H, num_calls, d_var, var_bins, d_t2, sz0, sz1, d_bw):
        _chk(self.lib.pb_bus_apply(self.h, handle, C.c_void_p(d_trace_ptr), C.c_size_t(H), C.c_int(num_calls), C.c_void_p(d_var), C.c_size_t(var_bins),
                                   C.c_void_p(d_t2), C.c_uint32(sz0), C.c_uint32(sz1), C.c_void_p(d_bw)), "pb_bus_apply")

    def bus_free(self, handle):
        self.lib.pb_bus_free(handle)

    # ---- stage 0 (reference symbols) ----
    def apc_tracegen(self, d_out_ptr, H, d_airs_ptr, d_subs_ptr, n_subs, num_calls):
        _chk(self.lib._apc_tracegen(C.c_void_p(d_out_ptr), C.c_size_t(H), C.c_void_p(d_airs_ptr), C.c_void_p(d_subs_ptr),
                                    C.c_size_t(n_subs), C.c_int(num_calls)), "_apc_tracegen")

    def apc_apply_derived_expr(self, d_out_ptr, H, num_calls, d_specs_ptr, n_cols, d_bc_ptr):
        _chk(self.lib._apc_apply_derived_expr(C.c_void_p(d_out_ptr), C.c_size_t(H), C.c_int(num_calls), C.c_void_p(d_specs_ptr),
                                              C.c_size_t(n_cols), C.c_void_p(d_bc_ptr)), "_apc_apply_derived_expr")

    def apc_apply_bus(self, d_out_ptr, num_calls, d_bc_ptr, bc_len, d_ints_ptr, n_ints, d_spans_ptr, n_spans, var_bus, d_var, var_bins,
                      t2_bus, d_t2, sz0, sz1, bw_bus, d_bw):
        _chk(self.lib._apc_apply_bus(C.c_void_p(d_out_ptr), C.c_int(num_calls), C.c_void_p(d_bc_ptr), C.c_size_t(bc_len),
                                     C.c_void_p(d_ints_ptr), C.c_size_t(n_ints), C.c_void_p(d_spans_ptr), C.c_size_t(n_spans),
                                     C.c_uint32(var_bus), C.c_void_p(d_var), C.c_size_t(var_bins), C.c_uint32(t2_bus), C.c_void_p(d_t2),
                                     C.c_uint32(sz0), C.c_uint32(sz1), C.c_uint32(bw_bus), C.c_void_p(d_bw)), "_apc_apply_bus")


class Group:
    """pb_group_t: contexts that prove as the ranks of one process (pb_prove_chips_group).  The library runs one thread per rank and
    exchanges device to device; rank r = ctxs[r].  The contexts stay the caller's: close the group before them."""

    def __init__(self, ctxs):
        self.lib = load_library()
        self.ctxs = list(ctxs)
        self.world = len(self.ctxs)
        arr = (C.c_void_p * max(1, self.world))(*[c.h.value for c in self.ctxs])
        h = C.c_void_p()
        _chk(self.lib.pb_group_create(arr, C.c_int(self.world), C.byref(h)), "pb_group_create")
        self.h = h
        self._chips = None

    def close(self):
        if self.h:
            self.lib.pb_group_destroy(self.h)
            self.h = None

    def prove_chips(self, chips, want_queries=True):
        """chips[r]: rank r's [(Air, d_trace_ptr, log_n, width)] as Context.prove_chips_sharded takes them (d_trace_ptr: rank r's column
        block on its context's device, 0 when empty).  -> the tuple of Context.prove_chips.  Ranks with different numbers of chips are
        refused here with PB_ERR_INVALID_ARG: the C call takes one n_chips for all of them."""
        if len(chips) != self.world:
            raise ValueError("one list of chips per rank: %d ranks, %d lists" % (self.world, len(chips)))
        K = len(chips[0])
        if any(len(c) != K for c in chips):
            raise PbError(PB_ERR_INVALID_ARG, "pb_prove_chips_group (n_chips differs between ranks)")
        arrs = [(Chip * max(1, K))(*[Chip(a.h.value if a else None, int(p or 0), int(ln), int(w)) for a, p, ln, w in c]) for c in chips]
        ptrs = (C.c_void_p * self.world)(*[C.addressof(a) for a in arrs])
        proof = ChipsProof()
        cums = np.zeros((K, 4), dtype=np.uint32)
        _chk(self.lib.pb_prove_chips_group(self.h, ptrs, C.c_size_t(K), C.byref(proof), cums.ctypes.data_as(C.c_void_p)), "pb_prove_chips_group")
        self._chips = (arrs[0], K)
        ys, q = self.query_chips(want_queries)
        return proof.as_dict(), cums, ys, q

    def query_chips(self, want_queries=True):
        """opened values and query openings of the group's last proof (pb_query_chips_group); its AIRs and traces must still be alive"""
        if self._chips is None:
            raise PbError(PB_ERR_INVALID_ARG, "pb_query_chips_group (no proof of this group)")
        arr, K = self._chips
        n_open, wpq = C.c_size_t(), C.c_size_t()
        _chk(self.lib.pb_chips_sizes(arr, C.c_size_t(K), C.byref(n_open), C.byref(wpq)), "pb_chips_sizes")
        nq = self.ctxs[0].n_queries
        ys = np.empty((n_open.value, 4), dtype=np.uint32)
        q = np.empty((nq, wpq.value), dtype=np.uint32) if want_queries and nq else None
        _chk(self.lib.pb_query_chips_group(self.h, q.ctypes.data_as(C.c_void_p) if q is not None else None, C.c_size_t(q.size if q is not None else 0),
                                           ys.ctypes.data_as(C.c_void_p), C.c_size_t(ys.size)), "pb_query_chips_group")
        return ys, q
