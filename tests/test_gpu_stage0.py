"""Stage 0 against a plain restatement of the reference kernels: the gather (_apc_tracegen), the derived columns
(_apc_apply_derived_expr) and the periphery histograms of both the drop-in _apc_apply_bus and the generated pb_bus_apply,
at the shapes where they split (grid-y launches, NVRTC modules, ragged interaction groups), at the edges of every table,
and with arguments outside the tables, which are counted nowhere (INTEGRATION.md §1).

The restatement below is numpy over rows: Python-int / uint64 arithmetic mod P for field values, histograms summed in uint64
and wrapped to u32 at the end, as the device's u32 atomics wrap.  It does not call the C oracle; the CPU tests pin it to the
oracle's line-by-line mirror of the reference (oracle/air.c) on in-table inputs, and check the oracle's out-of-table rule."""
import ctypes as C

import numpy as np
import pytest

from util import P, rand_field

PUSH_APC, PUSH_CONST, ADD, SUB, MUL, NEG, INV_OR_ZERO = range(7)
STACK = 16
VAR_BUS, T2_BUS, BW_BUS = 3, 7, 6
VAR_BINS, SZ0, SZ1 = 1 << 18, 256, 2048
BW_BINS = 1 << 17
SENTINEL = 0xA5A5A5A5
GUARD = 4096                    # words of sentinel on each side of every device histogram


# ---------------------------------------------------------------------------------------------------------------------
# the restatement

def _inv(a):
    """a^(P-2) mod P elementwise (so 0 -> 0: INV_OR_ZERO)"""
    r, b, e = np.ones_like(a), a.copy(), P - 2
    while e:
        if e & 1:
            r = r * b % P
        b = b * b % P
        e >>= 1
    return r


def ref_eval(bc, off, n, flat, rows):
    """the stack machine: canonical uint64 value of bc[off:off+n] at each of `rows`; PUSH_APC u reads flat[u + row]"""
    st, ip = [], off
    while ip < off + n:
        op = int(bc[ip])
        ip += 1
        if op in (PUSH_APC, PUSH_CONST):
            u = int(bc[ip])
            ip += 1
            st.append(flat[u + rows].astype(np.uint64) if op == PUSH_APC else np.full(rows.shape, u % P, dtype=np.uint64))
            assert len(st) <= STACK
        elif op in (ADD, SUB, MUL):
            b, a = st.pop(), st.pop()
            st.append((a + b) % P if op == ADD else (a + P - b) % P if op == SUB else a * b % P)
        elif op == NEG:
            st.append((P - st.pop()) % P)
        elif op == INV_OR_ZERO:
            st.append(_inv(st.pop()))
        else:
            raise ValueError("opcode %d" % op)
    assert len(st) == 1
    return st[0]


def ref_tracegen(out, airs, subs, num_calls):
    """apc_tracegen.cu: out[apc_col, r] = buffer[col * height + row + r * row_block_size] for r < num_calls, 0 for the other
    rows; columns without a substitution stay as they are.  out: (width, H) canonical, updated in place.
    airs: [(array (w, h), row_block_size)]; subs: [(air_index, col, row, apc_col)]"""
    H = out.shape[1]
    rows = np.arange(min(max(num_calls, 0), H))
    s = np.asarray(subs, dtype=np.int64).reshape(-1, 4)
    for ai, (a, rbs) in enumerate(airs):
        mine = s[s[:, 0] == ai]
        if not len(mine):
            continue
        src = (mine[:, 1] * a.shape[1] + mine[:, 2])[:, None] + rows[None, :] * rbs
        out[mine[:, 3], :len(rows)] = a.reshape(-1)[src]
        out[mine[:, 3], len(rows):] = 0
    return out


def ref_derived(out, num_calls, specs, bc):
    """apc_apply_derived_expr_kernel: specs [(col, off, len)] in order, each column = its expression on rows < num_calls (reading
    earlier derived columns of the same row), 0 below.  out: (width, H) canonical, in place; PUSH_APC operands are col * H."""
    H = out.shape[1]
    flat = out.reshape(-1)
    rows = np.arange(min(max(num_calls, 0), H))
    for col, off, n in specs:
        v = np.zeros(H, dtype=np.uint32)
        v[:len(rows)] = ref_eval(bc, off, n, flat, rows)
        out[col] = v
    return out


def ref_bus(trace, num_calls, bc, ints, spans, init=None):
    """apc_apply_bus_kernel with the out-of-table rule: -> (var, tuple2, bitwise) u32 histograms added onto `init`.
      variable range [value, max_bits]   bin 2^max_bits + value - 1   iff max_bits < 32, value < 2^max_bits, 2^(max_bits+1) - 1 <= bins
      tuple range    [v0, v1]            bin v0 * sz1 + v1            iff v0 < sz0 and v1 < sz1
      bitwise        [x, y, _, sel]      bin sel * 2^16 + x * 2^8 + y iff x < 256, y < 256, sel <= 1
    trace: (width, H) canonical; bytecode in the absolute-offset convention (compile_bus(machine, H))."""
    flat = np.ascontiguousarray(trace, dtype=np.uint32).reshape(-1)
    acc = [np.zeros(VAR_BINS, np.uint64), np.zeros(SZ0 * SZ1, np.uint64), np.zeros(BW_BINS, np.uint64)]
    rows = np.arange(max(num_calls, 0))
    for bus, _, a0 in ints:
        if bus not in (VAR_BUS, T2_BUS, BW_BUS):
            continue

        def arg(k):
            return ref_eval(bc, spans[a0 + k][0], spans[a0 + k][1], flat, rows)
        m = arg(0)
        if bus == VAR_BUS:
            v, b = arg(1), arg(2)
            one = np.uint64(1) << np.minimum(b, np.uint64(40))
            ok = (b < 32) & (v < one) & (2 * one - 1 <= VAR_BINS)
            k, idx = 0, one + v - 1
        elif bus == T2_BUS:
            v0, v1 = arg(1), arg(2)
            ok = (v0 < SZ0) & (v1 < SZ1)
            k, idx = 1, v0 * SZ1 + v1
        else:
            x, y, sel = arg(1), arg(2), arg(4)
            ok = (x < 256) & (y < 256) & (sel <= 1)
            k, idx = 2, sel * 65536 + x * 256 + y
        ok &= m != 0
        np.add.at(acc[k], idx[ok].astype(np.int64), m[ok])
    if init is not None:
        acc = [a + i.astype(np.uint64) for a, i in zip(acc, init)]
    return tuple((a & np.uint64(0xFFFFFFFF)).astype(np.uint32) for a in acc)


# ---------------------------------------------------------------------------------------------------------------------
# hand-written bytecode (the reference's encoding; constants are NOT reduced, so words >= P reach the kernels)

def e_col(c, H):
    return [PUSH_APC, c * H]


def e_const(u):
    return [PUSH_CONST, u]


def e_bin(a, op, b):
    return a + b + [op]


def derived_program(H):
    """columns 0..3 inputs; 4..10 derived, in order, each reading earlier ones: -> (width, specs [(col, off, len)], bytecode)"""
    exprs = [
        (4, [PUSH_APC, 0 * H, INV_OR_ZERO]),                                                   # inv(c0), c0 has 0 and P-1 rows
        (5, e_bin(e_bin(e_col(4, H), MUL, e_col(1, H)), ADD, e_const(P))),                      # d4 * c1 + P
        (6, e_bin(e_bin(e_col(5, H), SUB, e_col(2, H)), MUL, [PUSH_APC, 4 * H, INV_OR_ZERO])),  # (d5 - c2) * inv(d4)
        (7, e_bin(e_const(P + 1), ADD, e_const(0xFFFFFFFF))),                                  # 1 + (2^32 - 1 mod P)
        (8, [PUSH_APC, 3 * H, NEG, INV_OR_ZERO, NEG]),                                           # -inv(-c3), c3 has 1 and P-1 rows
    ]
    # all 16 stack slots: x0 - (x1 * (x2 + (x3 - ... (x14 * x15))))
    leaves = [e_col(i % 8, H) if i % 3 else e_const([0xFFFFFFFF, P, P + 1, 7][i % 4]) for i in range(STACK)]
    deep = []
    for x in leaves:
        deep += x
    for i in range(STACK - 1, 0, -1):
        deep.append([SUB, MUL, ADD][i % 3])
    exprs.append((9, deep))
    exprs.append((10, e_bin(e_col(9, H), MUL, e_col(6, H))))
    bc, specs = [], []
    for col, code in exprs:
        specs.append((col, len(bc), len(code)))
        bc += code
    return 11, specs, bc


def derived_inputs(rng, H):
    base = rand_field(rng, (11, H))
    base[0, 0::5], base[0, 1::5] = 0, P - 1                  # INV_OR_ZERO of 0 and of P-1
    base[3, 0::2], base[3, 1::4] = 1, P - 1
    base[2, 2::7] = base[1, 2::7]
    return base


def keccak_shape_machine():
    """the bench's AIR (bench.py machine_for at the defaults: synthetic_machine(2022, 187) + synthetic_bus(1734), same seeds)"""
    from powdr_b200 import machine as M
    base = M.synthetic_machine(2022, 187, seed=0xB2000001)
    return M.SymbolicMachine(base.constraints, M.synthetic_bus(base, 1734, seed=0xB2000002))


def n_periphery(mach):
    return sum(1 for b in mach.bus_interactions if b["id"] in (VAR_BUS, T2_BUS, BW_BUS))


def in_table_machine(n_cols=48, n_ints=300, seed=11):
    """a bus whose periphery arguments are all inside their tables on the trace of in_table_trace: columns 0..15 bytes,
    16..23 values < 2^11, 24..31 multiplicities in [0, 4) or P - [0, 4), 32..47 17-bit values"""
    rng = np.random.default_rng(seed)
    c = lambda i: "c%d@%d" % (i, i)
    ints = []
    for i in range(n_ints):
        t = i % 5
        mult = [1, c(24 + i % 8), ["-", c(24 + i % 8)], 1 << 20, P - 1][int(rng.integers(0, 5))]
        if t == 0:
            ints.append({"id": VAR_BUS, "mult": mult, "args": [c(32 + i % 16), int(rng.integers(17, 18))]})
        elif t == 1:
            ints.append({"id": VAR_BUS, "mult": mult, "args": [c(i % 16), int(rng.integers(8, 18))]})
        elif t == 2:
            ints.append({"id": T2_BUS, "mult": mult, "args": [c(i % 16), c(16 + i % 8)]})
        elif t == 3:
            ints.append({"id": BW_BUS, "mult": mult, "args": [c(i % 16), c((i + 5) % 16), 0, int(i % 2)]})
        else:
            ints.append({"id": 1, "mult": mult, "args": [c(i % n_cols), 7]})     # memory bus: not a periphery table
    return ints, n_cols


def in_table_trace(rng, H, n_cols=48):
    tr = np.zeros((n_cols, H), dtype=np.uint32)
    tr[0:16] = rng.integers(0, 256, (16, H))
    tr[16:24] = rng.integers(0, SZ1, (8, H))
    m = rng.integers(0, 4, (8, H)).astype(np.uint32)
    tr[24:32] = m
    tr[32:48] = rng.integers(0, 1 << 17, (16, H))
    return tr


def edge_machine():
    """in-table edges: value = 2^b - 1 for b = 0..17, x = y = 255 under both selectors, the tuple (sz0 - 1, sz1 - 1); the
    multiplicity column m cycles through 1, 2^20 and P-1 and is 0 on every other lane"""
    c = lambda i: "c%d@%d" % (i, i)
    M_, V, B, X, T0, T1 = 0, 1, 2, 3, 4, 5
    ints = []
    for b in range(18):
        ints.append({"id": VAR_BUS, "mult": c(M_), "args": [(1 << b) - 1, b]})
    ints.append({"id": VAR_BUS, "mult": c(M_), "args": [c(V), c(B)]})         # per row: (2^(r mod 18) - 1, r mod 18)
    for sel in (0, 1):
        ints.append({"id": BW_BUS, "mult": c(M_), "args": [255, 255, 0, sel]})
        ints.append({"id": BW_BUS, "mult": 1, "args": [c(X), c(X), 0, sel]})    # x = y = 255 on every row: one bin per warp
    ints.append({"id": T2_BUS, "mult": c(M_), "args": [SZ0 - 1, SZ1 - 1]})
    ints.append({"id": T2_BUS, "mult": c(M_), "args": [c(T0), c(T1)]})
    ints.append({"id": VAR_BUS, "mult": 1, "args": [0, 0]})                  # all lanes, bin 0
    return ints, 6


def edge_trace(rng, H):
    tr = np.zeros((6, H), dtype=np.uint32)
    r = np.arange(H)
    tr[0] = np.where(r % 2 == 0, np.array([1, 1 << 20, P - 1], dtype=np.uint32)[(r // 2) % 3], 0)
    tr[1] = (1 << (r % 18)) - 1
    tr[2] = r % 18
    tr[3] = 255
    tr[4], tr[5] = SZ0 - 1, SZ1 - 1
    return tr


def out_of_table_machine():
    """every kind of argument outside its table, next to in-table neighbours (the bins they would alias into)"""
    c = lambda i: "c%d@%d" % (i, i)
    ints = []
    for b in range(18, 41):                                                 # max_bits beyond the table
        ints.append({"id": VAR_BUS, "mult": 1, "args": [b % 7, b]})
    ints.append({"id": VAR_BUS, "mult": 1, "args": [0, 0xFFFFFFFF]})          # a max_bits word >= P (reduced: 268435453)
    ints.append({"id": VAR_BUS, "mult": c(0), "args": [c(1), c(2)]})          # per row: (r mod 6, 18 + r mod 23)
    for b in range(18):
        ints.append({"id": VAR_BUS, "mult": 1, "args": [1 << b, b]})          # value = 2^b would be (0, b + 1)
    ints.append({"id": VAR_BUS, "mult": 1, "args": [P - 1, 17]})
    ints.append({"id": VAR_BUS, "mult": 1, "args": [P - 1, 31]})
    for x, y, sel in [(256, 3, 0), (300, 5, 0), (511, 255, 0), (3, 256, 1), (0, 0, 2), (0, 0, P - 1), (P - 1, 0, 0)]:
        ints.append({"id": BW_BUS, "mult": 1, "args": [x, y, 0, sel]})
    ints.append({"id": BW_BUS, "mult": 1, "args": [c(3), c(4), 0, c(5)]})     # per row: x in [256, 512), selector 0
    wrap = (1 << 32) // SZ1                                                 # v0 * sz1 wraps to 0 in u32
    for v0, v1 in [(0, SZ1), (1, SZ1 + 5), (SZ0, 0), (wrap + 3, 17), (wrap, 0), (P - 1, 1), (2, P - 1)]:
        ints.append({"id": T2_BUS, "mult": 1, "args": [v0, v1]})
    ints.append({"id": T2_BUS, "mult": 1, "args": [c(6), c(7)]})              # per row: a wrapped v0
    # the in-table neighbours
    ints += [{"id": VAR_BUS, "mult": 1, "args": [0, b]} for b in range(18)]
    ints += [{"id": BW_BUS, "mult": 1, "args": [0, 3, 0, 1]}, {"id": BW_BUS, "mult": 1, "args": [1, 5, 0, 1]}]
    ints += [{"id": T2_BUS, "mult": 1, "args": [1, 0]}, {"id": T2_BUS, "mult": 1, "args": [3, 17]}, {"id": T2_BUS, "mult": 1, "args": [0, 0]}]
    return ints, 8


def out_of_table_trace(rng, H):
    tr = np.zeros((8, H), dtype=np.uint32)
    r = np.arange(H)
    tr[0] = 1 + r % 3
    tr[1], tr[2] = r % 6, 18 + r % 23
    tr[3], tr[4], tr[5] = 256 + r % 256, r % 256, 0
    tr[6], tr[7] = (1 << 32) // SZ1 + r % 8, r % 64
    return tr


def _machine(ints, n_cols):
    from powdr_b200 import machine as M
    # every column referenced, so that column i is index i
    pad = [{"id": 1, "mult": 0, "args": ["c%d@%d" % (i, i) for i in range(n_cols)]}]
    return M.SymbolicMachine([], ints + pad)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the restatement against the oracle, the oracle's out-of-table rule, and the 970-interaction generated kernel

def test_restated_gather_matches_oracle(orc):
    rng = np.random.default_rng(1)
    H = 64
    airs = [(rand_field(rng, (5, 2 * H + 1)), 1), (rand_field(rng, (4, 3 * 2 * H)), 3), (rand_field(rng, (6, 7 * 2 * H)), 7)]
    subs = [(0, 4, 1, 0), (1, 0, 2, 2), (2, 5, 6, 3), (2, 0, 0, 5), (1, 3, 0, 6), (0, 0, 0, 8)]
    for n in (0, 1, 31, H - 1, H, 2 * H):
        exp = orc.apc_tracegen(H, 9, airs, subs, n)
        got = ref_tracegen(np.full((9, H), 0xDEADBEEF % P, dtype=np.uint32), airs, subs, n)
        assert (got == exp).all(), n


def test_restated_derived_columns_match_oracle(orc):
    rng = np.random.default_rng(2)
    H = 128
    width, specs, bc = derived_program(H)
    base = derived_inputs(rng, H)
    for n in (0, 1, 100, H):
        exp = orc.apc_apply_derived(base.copy(), n, specs, bc)
        got = ref_derived(base.copy(), n, specs, bc)
        assert (got == exp).all(), n
    assert (exp[7] == (P + 1 + 0xFFFFFFFF) % P).all()            # n = H: constants P + 1 and 2^32 - 1 reduced mod P


@pytest.mark.parametrize("case", ["in_table", "edges", "out_of_table"])
def test_restated_histograms_match_oracle(orc, case):
    from powdr_b200 import machine as M
    rng = np.random.default_rng(3)
    H = 256
    ints, n_cols = {"in_table": in_table_machine, "edges": edge_machine, "out_of_table": out_of_table_machine}[case]()
    tr = {"in_table": in_table_trace, "edges": edge_trace, "out_of_table": out_of_table_trace}[case](rng, H)
    mach = _machine(ints, n_cols)
    ib, isp, ibc = M.compile_bus(mach, H)
    exp = orc.apc_apply_bus(tr, H - 3, ibc, ib, isp, (VAR_BUS, VAR_BINS), (T2_BUS, SZ0, SZ1), BW_BUS)
    got = ref_bus(tr, H - 3, ibc, ib, isp)
    for g, e, name in zip(got, exp, ("var", "tuple2", "bitwise")):
        assert (g == e).all(), name
    if case == "out_of_table":
        # only the in-table neighbours count: one per row in each of their bins, nothing anywhere else
        n = H - 3
        var_bins = {(1 << b) - 1 for b in range(18)}
        assert set(np.flatnonzero(got[0])) == var_bins and (got[0][sorted(var_bins)] == n).all()
        assert set(np.flatnonzero(got[1])) == {SZ1, 3 * SZ1 + 17, 0} and set(got[1][[SZ1, 3 * SZ1 + 17, 0]]) == {n}
        assert set(np.flatnonzero(got[2])) == {65536 + 3, 65536 + 256 + 5}


def test_generated_periphery_kernel_compiles_at_the_keccak_shape():
    """970 periphery interactions: 61 generated functions of 16 (the last of 10) in 8 NVRTC modules of 128 (the last of 74),
    compiled for sm_90a with no device (ctx = out = NULL)"""
    import powdr_b200
    from powdr_b200 import capi, machine as M
    lib = powdr_b200.load_library()
    mach = keccak_shape_machine()
    n = n_periphery(mach)
    assert (n, -(-n // 16), n % 16, -(-n // 128), n % 128) == (970, 61, 10, 8, 74)
    ints, isp, ibc = M.compile_bus(mach, 1)
    ibc = np.array(ibc, dtype=np.uint32)
    spn = (capi.Span * len(isp))()
    for i, (o, l) in enumerate(isp):
        spn[i].off, spn[i].len = o, l
    di = (capi.DevInteraction * len(ints))()
    for i, (b, k, o) in enumerate(ints):
        di[i].bus_id, di[i].num_args, di[i].args_index_off = b, k, o
    assert lib.pb_bus_compile(None, ibc.ctypes.data_as(C.c_void_p), C.c_size_t(ibc.size), spn, C.c_size_t(len(isp)), di, C.c_size_t(len(ints)),
                              C.c_uint32(mach.width), C.c_uint32(VAR_BUS), C.c_uint32(T2_BUS), C.c_uint32(BW_BUS), None) == 0


# ---------------------------------------------------------------------------------------------------------------------
# GPU

def _upload_structs(ctx, arr):
    raw = np.frombuffer(bytes(arr), dtype=np.uint8)
    return ctx.alloc(raw.nbytes).upload(raw)


def _gather(ctx, out_init, airs, subs, num_calls):
    """_apc_tracegen on the device (cells raw, as the kernel copies words) -> (device output, restated output)"""
    from powdr_b200 import capi
    keep = [ctx.to_device(a, monty=False) for a, _ in airs]
    A = (capi.OriginalAir * len(airs))()
    for i, ((a, rbs), d) in enumerate(zip(airs, keep)):
        A[i].width, A[i].height, A[i].buffer, A[i].row_block_size = a.shape[0], a.shape[1], d.ptr, rbs
    S = (capi.Subst * len(subs))()
    for i, s in enumerate(subs):
        S[i].air_index, S[i].col, S[i].row, S[i].apc_col = (int(x) for x in s)
    d_airs, d_subs = _upload_structs(ctx, A), _upload_structs(ctx, S)
    d_out = ctx.to_device(out_init, monty=False)
    ctx.apc_tracegen(d_out.ptr, out_init.shape[1], d_airs.ptr, d_subs.ptr, len(subs), num_calls)
    ctx.synchronize()
    got = d_out.download(out_init.shape)
    return got, ref_tracegen(out_init.copy(), airs, subs, num_calls)


@pytest.mark.gpu
def test_gather_70000_substitutions_two_grid_y_launches(ctx):
    rng = np.random.default_rng(10)
    H, n_subs = 32, 70000
    airs = [(rand_field(rng, (300, H)), 1), (rand_field(rng, (40, 3 * H)), 3)]
    ai = rng.integers(0, 2, n_subs)
    col = np.where(ai == 0, rng.integers(0, 300, n_subs), rng.integers(0, 40, n_subs))
    row = np.where(ai == 0, 0, rng.integers(0, 3, n_subs))
    subs = np.stack([ai, col, row, rng.permutation(n_subs + 7)[:n_subs]], axis=1)
    init = np.full((n_subs + 7, H), SENTINEL, dtype=np.uint32)
    got, exp = _gather(ctx, init, airs, subs, H - 5)
    assert (got == exp).all()
    assert (got[subs[65535:, 3]] != SENTINEL).all()          # the second launch's substitutions were written


@pytest.mark.gpu
@pytest.mark.parametrize("calls", ["0", "1", "31", "H-1", "H", "2H"])
def test_gather_row_blocks_and_call_counts(ctx, calls):
    rng = np.random.default_rng(11)
    H = 2048
    n = {"0": 0, "1": 1, "31": 31, "H-1": H - 1, "H": H, "2H": 2 * H}[calls]
    hh = 2 * H
    airs = [(rand_field(rng, (6, hh)), 1), (rand_field(rng, (5, 3 * hh)), 3), (rand_field(rng, (4, 7 * hh)), 7)]
    subs = [(0, 5, 0, 0), (1, 4, 2, 1), (2, 3, 6, 2), (2, 0, 0, 4), (1, 0, 1, 5), (0, 0, 0, 7), (2, 1, 3, 9), (1, 2, 2, 10)]
    init = np.full((12, H), SENTINEL, dtype=np.uint32)        # columns 3, 6, 8, 11 are not substituted: they come back untouched
    got, exp = _gather(ctx, init, airs, subs, n)
    assert (got == exp).all()
    assert (got[[3, 6, 8, 11]] == SENTINEL).all()


@pytest.mark.gpu
def test_gather_at_2p20_rows(ctx):
    rng = np.random.default_rng(12)
    H = 1 << 20
    airs = [(rand_field(rng, (3, H)), 1), (rand_field(rng, (2, 3 * H)), 3)]
    subs = [(0, 2, 0, 0), (1, 1, 2, 1), (1, 0, 0, 3), (0, 0, 0, 4)]
    init = np.full((5, H), SENTINEL, dtype=np.uint32)
    got, exp = _gather(ctx, init, airs, subs, H - 3)
    assert (got == exp).all()


@pytest.mark.gpu
@pytest.mark.parametrize("H,num_calls", [(1024, 700), (1024, 1024), (256, 0)])
def test_derived_columns(ctx, H, num_calls):
    """a chain of derived columns reading earlier ones, INV_OR_ZERO of 0 and P-1, constants P, P+1 and 2^32-1, an expression
    that fills all 16 stack slots, zero fill below num_calls"""
    from powdr_b200 import capi
    rng = np.random.default_rng(13 + H + num_calls)
    width, specs, bc = derived_program(H)
    base = derived_inputs(rng, H)
    exp = ref_derived(base.copy(), num_calls, specs, bc)
    d_out = ctx.to_device(base)
    D = (capi.DerivedExprSpec * len(specs))()
    for i, (c, o, l) in enumerate(specs):
        D[i].col_base, D[i].span.off, D[i].span.len = c * H, o, l
    d_specs = _upload_structs(ctx, D)
    d_bc = ctx.to_device(np.array(bc, dtype=np.uint32), monty=False)
    ctx.apc_apply_derived_expr(d_out.ptr, H, num_calls, d_specs.ptr, len(specs), d_bc.ptr)
    ctx.synchronize()
    got = ctx.to_host(d_out, base.shape)
    assert (got == exp).all()
    assert not got[4:, num_calls:].any()


class _Hists:
    """the three device histograms, each inside a guard region of sentinel words that must come back unchanged"""

    def __init__(self, ctx, init):
        self.ctx, self.init = ctx, init
        self.bufs = []
        for h in init:
            raw = np.full(h.size + 2 * GUARD, SENTINEL, dtype=np.uint32)
            raw[GUARD:GUARD + h.size] = h
            self.bufs.append(ctx.alloc(raw.nbytes).upload(raw))
        self.var, self.t2, self.bw = (b.ptr + 4 * GUARD for b in self.bufs)

    def read(self):
        self.ctx.synchronize()
        out = []
        for b, h in zip(self.bufs, self.init):
            raw = b.download(h.size + 2 * GUARD)
            assert (raw[:GUARD] == SENTINEL).all() and (raw[GUARD + h.size:] == SENTINEL).all(), "write outside a histogram"
            out.append(raw[GUARD:GUARD + h.size])
        return out


def _both_paths(ctx, mach, trace, num_calls, init=None):
    """the histograms of _apc_apply_bus and of pb_bus_apply, each on fresh guarded buffers starting at `init`, against ref_bus"""
    from powdr_b200 import capi, machine as M
    H = trace.shape[1]
    if init is None:
        init = (np.zeros(VAR_BINS, np.uint32), np.zeros(SZ0 * SZ1, np.uint32), np.zeros(BW_BINS, np.uint32))
    ints, spans, bc = M.compile_bus(mach, H)
    exp = ref_bus(trace, num_calls, bc, ints, spans, init)
    d_tr = ctx.to_device(trace)
    d_bc = ctx.to_device(np.array(bc, dtype=np.uint32), monty=False)
    I = (capi.DevInteraction * len(ints))()
    for i, (b, n, o) in enumerate(ints):
        I[i].bus_id, I[i].num_args, I[i].args_index_off = b, n, o
    SP = (capi.Span * len(spans))()
    for i, (o, l) in enumerate(spans):
        SP[i].off, SP[i].len = o, l
    d_i, d_s = _upload_structs(ctx, I), _upload_structs(ctx, SP)
    h = _Hists(ctx, init)
    ctx.apc_apply_bus(d_tr.ptr, num_calls, d_bc.ptr, len(bc), d_i.ptr, len(ints), d_s.ptr, len(spans), VAR_BUS, h.var, VAR_BINS,
                      T2_BUS, h.t2, SZ0, SZ1, BW_BUS, h.bw)
    dropin = h.read()
    handle = ctx.bus_compile(M.compile_bus(mach, 1), mach.width, VAR_BUS, T2_BUS, BW_BUS)
    try:
        h = _Hists(ctx, init)
        ctx.bus_apply(handle, d_tr.ptr, H, num_calls, h.var, VAR_BINS, h.t2, SZ0, SZ1, h.bw)
        generated = h.read()
    finally:
        ctx.bus_free(handle)
    for path, got in (("_apc_apply_bus", dropin), ("pb_bus_apply", generated)):
        for g, e, name in zip(got, exp, ("var", "tuple2", "bitwise")):
            bad = np.flatnonzero(g != e)
            assert not len(bad), "%s %s histogram: bins %s = %s, expected %s" % (path, name, bad[:8], g[bad[:8]], e[bad[:8]])
    return exp


@pytest.mark.gpu
def test_histograms_keccak_shape(ctx):
    """the bench's AIR at 2^12 rows with byte-valued cells: 970 periphery interactions, so pb_bus_apply runs 8 modules and a
    ragged last group; the negated-column multiplicities are P - c"""
    mach = keccak_shape_machine()
    assert n_periphery(mach) == 970
    rng = np.random.default_rng(0xB2000007)
    H = 1 << 12
    tr = rng.integers(0, 256, (mach.width, H)).astype(np.uint32)
    var, t2, bw = _both_paths(ctx, mach, tr, H)
    assert var.any() and bw[:65536].any() and bw[65536:].any()


@pytest.mark.gpu
def test_histograms_more_than_128_in_table_interactions(ctx):
    ints, n_cols = in_table_machine()
    mach = _machine(ints, n_cols)
    assert n_periphery(mach) > 128
    rng = np.random.default_rng(14)
    H = 1024
    tr = in_table_trace(rng, H, n_cols)
    tr[:, 1000:] = rand_field(rng, (n_cols, 24))              # garbage past num_apc_calls
    var, t2, bw = _both_paths(ctx, mach, tr, 1000)
    # every interaction is in its table: each counts once per row with a non-zero multiplicity
    assert var.any() and t2.any() and bw[:65536].any() and bw[65536:].any()


@pytest.mark.gpu
@pytest.mark.parametrize("num_calls", [1, 33, 127, 129, 256])
def test_histograms_in_table_edges(ctx, num_calls):
    """2^b - 1 for every b, x = y = 255 under both selectors, (sz0 - 1, sz1 - 1), multiplicities 1, 2^20 and P-1 on every other
    lane; all lanes of a warp on one bin; rows past num_apc_calls hold garbage"""
    ints, n_cols = edge_machine()
    mach = _machine(ints, n_cols)
    rng = np.random.default_rng(15)
    H = 256
    tr = edge_trace(rng, H)
    tr[:, num_calls:] = rand_field(rng, (n_cols, H - num_calls))
    var, t2, bw = _both_paths(ctx, mach, tr, num_calls)
    assert var[(1 << 18) - 2] and bw[65535] and bw[131071] and t2[-1]        # the last bin of every table


@pytest.mark.gpu
def test_histograms_out_of_table_arguments_are_counted_nowhere(ctx):
    """max_bits 18..40 and >= P, value = 2^b, bitwise x or y >= 256 and selectors 2 and P-1, tuple v1 >= sz1, v0 >= sz0 and a
    v0 * sz1 that wraps in u32: none counts, the in-table neighbours they would alias into count once per row"""
    ints, n_cols = out_of_table_machine()
    mach = _machine(ints, n_cols)
    rng = np.random.default_rng(16)
    H = 512
    tr = out_of_table_trace(rng, H)
    var, t2, bw = _both_paths(ctx, mach, tr, H)
    assert var.sum() == 18 * H and t2.sum() == 3 * H and bw.sum() == 2 * H


@pytest.mark.gpu
def test_histograms_add_onto_non_zero_counts(ctx):
    ints, n_cols = in_table_machine(n_ints=150, seed=17)
    ints += edge_machine()[0][:4]
    mach = _machine(ints, n_cols)
    rng = np.random.default_rng(17)
    H = 512
    tr = in_table_trace(rng, H, n_cols)
    init = (rng.integers(0, 1 << 32, VAR_BINS, dtype=np.uint64).astype(np.uint32),
            rng.integers(0, 1 << 32, SZ0 * SZ1, dtype=np.uint64).astype(np.uint32),
            rng.integers(0, 1 << 32, BW_BINS, dtype=np.uint64).astype(np.uint32))
    _both_paths(ctx, mach, tr, H - 1, init)
