"""Generated AIRs for the code generators of stage 2 and the LogUp argument, and a plain evaluator of what they must compute.

The generators (air_jit.cuh, logup_jit.cuh, bus_jit.cuh) write different code for different expression shapes: literal folding,
Shoup products with the literal on either side, hoisted and load-at-use columns, group cuts at 600 ops, module cuts at 2000 words,
LogUp chunks of one, two and three or more interactions, literal multiplicities and literal arguments folded on the host.  The
cases below are built so that every one of those shapes occurs, at fixed seeds.

The evaluator works from the JSON trees (and, for OP_INV_OR_ZERO, which has no JSON form, from the raw words), vectorised over rows
in numpy uint64 with a reduction mod P after every operation.  It does not go through machine.emit_expr or the C oracle, so an
emission bug shared by the GPU and the oracle shows up against it."""
import numpy as np

from powdr_b200 import machine as M
from test_oracle_logup import e4, e4_mul

P = M.P
SHIFT = 31                                  # coset shift of the LDE (pb_quotient's default)
EDGE = [0, 1, 2, P - 1, P - 2, (P - 1) // 2, (P + 1) // 2, 1 << 27]
MODULE_WORDS = 2000                                          # air_jit.cuh
MODULE_CHUNKS = 16                                           # logup_jit.cuh
STACK = 16


def x(i):
    return "c%d@%d" % (i, i)


def _cid(ref):
    return int(ref.rsplit("@", 1)[1])


# ---------------------------------------------------------------- evaluator
def ops_of_tree(expr):
    """post-order op stream of a JSON tree; iterative, since a long sum chain nests thousands of levels deep"""
    out, work = [], [(expr, False)]
    while work:
        e, done = work.pop()
        if isinstance(e, int):
            out.append(("k", e % P))
        elif isinstance(e, str):
            out.append(("x", _cid(e)))
        elif len(e) == 3:
            if done:
                out.append((e[1],))
            else:
                work += [(e, True), (e[2], False), (e[0], False)]
        elif done:
            out.append(("neg",))
        else:
            work += [(e, True), (e[1], False)]
    return out


_WORD_OPS = {2: ("+",), 3: ("-",), 4: ("*",), 5: ("neg",), 6: ("inv",)}


def ops_of_words(words):
    """op stream of raw reference bytecode (PUSH_APC operand = column index)"""
    out, i = [], 0
    while i < len(words):
        op = words[i]
        if op in (M.OP_PUSH_APC, M.OP_PUSH_CONST):
            out.append(("x" if op == M.OP_PUSH_APC else "k", words[i + 1] if op == M.OP_PUSH_APC else words[i + 1] % P))
            i += 2
        else:
            out.append(_WORD_OPS[op])
            i += 1
    return out


def stack_depth(ops):
    d = best = 0
    for o in ops:
        d += 1 if o[0] in ("x", "k") else -1 if o[0] in ("+", "-", "*") else 0
        best = max(best, d)
    return best


def _inv(a):
    r, b, e = np.ones_like(a), a.copy(), P - 2
    while e:
        if e & 1:
            r = r * b % P
        b = b * b % P
        e >>= 1
    return r                                  # 0 -> 0


def eval_ops(ops, mat):
    """mat: (width, n) canonical -> (n,) uint64 values of the expression on every row"""
    n = mat.shape[1]
    st = []
    for o in ops:
        t = o[0]
        if t == "x":
            st.append(mat[o[1]].astype(np.uint64))
        elif t == "k":
            st.append(np.full(n, o[1], dtype=np.uint64))
        elif t == "neg":
            st.append((P - st.pop()) % P)
        elif t == "inv":
            st.append(_inv(st.pop()))
        else:
            b, a = st.pop(), st.pop()
            st.append((a + b) % P if t == "+" else (a + (P - b)) % P if t == "-" else a * b % P)
    assert len(st) == 1
    return st[0]


def alpha_fold(values, alpha):
    """values: per constraint (n,) arrays -> (4, n): sum_k alpha^(C-1-k) c_k"""
    C = len(values)
    n = values[0].shape[0] if C else 0
    out = np.zeros((4, n), dtype=np.uint64)
    pw = e4(1)
    for k in range(C - 1, -1, -1):
        for l in range(4):
            out[l] = (out[l] + values[k] * np.uint64(pw[l]) % P) % P
        pw = e4_mul(pw, [int(a) for a in alpha])
    return out.astype(np.uint32)


def quotient(fold, log_n, shift=SHIFT):
    """fold: (4, 2N) over the bit-reversed LDE rows -> (2, 4, N): the half r < N times (s^N - 1)^-1, the other (-s^N - 1)^-1"""
    n = 1 << log_n
    sn = pow(shift, n, P)
    z = [pow((sn - 1) % P, P - 2, P), pow((-sn - 1) % P, P - 2, P)]
    f = fold.astype(np.uint64)
    return np.stack([f[:, c * n:(c + 1) * n] * np.uint64(z[c]) % P for c in range(2)]).astype(np.uint32)


# Ext4 over rows: four (n,) uint64 limbs
def _v_mul(a, b):
    t = [0] * 7
    for i in range(4):
        for j in range(4):
            t[i + j] = (t[i + j] + a[i] * b[j] % P) % P
    return [(t[i] + 11 * (t[i + 4] if i + 4 < 7 else 0)) % P for i in range(4)]


def _v_inv(a):
    e = P ** 4 - 2
    r = [np.ones_like(a[0])] + [np.zeros_like(a[0]) for _ in range(3)]
    while e:
        if e & 1:
            r = _v_mul(r, a)
        a = _v_mul(a, a)
        e >>= 1
    return r


def chunk_starts(bus_json, max_degree=3):
    """greedy chunking in declaration order: a chunk stays while max(1, max_i(deg m_i - deg d_i)) + sum_i deg d_i <= 3
    (deg d_i = the largest argument degree).  None when one interaction alone breaks the bound."""
    starts, i, n = [], 0, len(bus_json)
    while i < n:
        starts.append(i)
        sum_dd = max_extra = cnt = 0
        while i < n:
            b = bus_json[i]
            md = M.degree(b["mult"])
            dd = max([M.degree(a) for a in b["args"]], default=0)
            nsum, nextra = sum_dd + dd, max(max_extra, md - dd if md > dd else 0)
            if max(1, nextra) + nsum > max_degree:
                if cnt == 0:
                    return None
                break
            sum_dd, max_extra = nsum, nextra
            i += 1
            cnt += 1
    return starts + [n]


def perm_trace(bus_json, trace, alpha_lu, beta_lu):
    """-> (perm (4*(chunks+1), N), cumulative sum [4], chunk starts): perm_c = sum_{i in c} m_i / d_i,
    d_i = alpha_lu + sum_j beta^j arg_j + beta^k (bus_i + 1), then the running sum over rows"""
    cs = chunk_starts(bus_json)
    n = trace.shape[1]
    al = [int(a) for a in alpha_lu]
    be = [int(a) for a in beta_lu]
    ms, ds = [], []
    for b in bus_json:
        ms.append(eval_ops(ops_of_tree(b["mult"]), trace))
        d = [np.full(n, al[l], dtype=np.uint64) for l in range(4)]
        bp = e4(1)
        for a in b["args"]:
            v = eval_ops(ops_of_tree(a), trace)
            d = [(d[l] + v * np.uint64(bp[l]) % P) % P for l in range(4)]
            bp = e4_mul(bp, be)
        last = e4_mul(bp, e4(int(b["id"]) + 1))
        ds.append([(d[l] + last[l]) % P for l in range(4)])
    k = len(bus_json)
    inv = _v_inv([np.concatenate([d[l] for d in ds]) for l in range(4)]) if k else None
    perm = np.zeros((4 * (len(cs)), n), dtype=np.uint64)
    for c in range(len(cs) - 1):
        for i in range(cs[c], cs[c + 1]):
            for l in range(4):
                perm[4 * c + l] = (perm[4 * c + l] + inv[l][i * n:(i + 1) * n] * ms[i] % P) % P
    nc = len(cs) - 1
    rows = perm[:4 * nc].reshape(nc, 4, n).sum(axis=0) % P if nc else np.zeros((4, n), dtype=np.uint64)
    perm[4 * nc:] = np.cumsum(rows, axis=1) % P
    return perm.astype(np.uint32), [int(v) for v in perm[4 * nc:, n - 1]], cs


# ---------------------------------------------------------------- generator
class Case:
    """One generated AIR: JSON constraints, raw-word constraints (OP_INV_OR_ZERO), bus interactions, over columns c0..c{width-1}."""

    def __init__(self, name, width, constraints=(), raw=(), bus=()):
        self.name, self.width = name, width
        self.constraints, self.raw, self.bus = list(constraints), list(raw), list(bus)
        used = set()
        for e in self.constraints + [b["mult"] for b in self.bus] + [a for b in self.bus for a in b["args"]]:
            used.update(_cid(r) for r in M.iter_refs(e))
        for w in self.raw:
            used.update(o[1] for o in ops_of_words(w) if o[0] == "x")
        missing = sorted(set(range(width)) - used)
        if missing:                              # every column is referenced, so column index = poly id
            self.constraints.append(_chain([x(i) for i in missing], 2 * len(missing) - 1))
        self.mach = M.SymbolicMachine(self.constraints, self.bus)
        assert self.mach.column_ids == list(range(width))

    def program(self):
        """(bytecode, spans) in the column-index convention: the JSON constraints, then the raw ones"""
        bc, spans = M.compile_constraints(self.mach)
        for w in self.raw:
            spans.append((len(bc), len(w)))
            bc = bc + list(w)
        return bc, spans

    def bus_program(self):
        return M.compile_bus(self.mach, 1) if self.bus else None

    def constraint_ops(self):
        return [ops_of_tree(c) for c in self.constraints] + [ops_of_words(w) for w in self.raw]

    def fold(self, mat, alpha):
        return alpha_fold([eval_ops(o, mat) for o in self.constraint_ops()], alpha)


def _chain(leaves, length, ops=("+", "-", "*")):
    """left-leaning chain over `leaves` (cycled) with exactly `length` packed instructions and stack depth 2"""
    steps = (length - 1) // 2
    e = leaves[0]
    for s in range(steps):
        e = [e, ops[s % len(ops)], leaves[(s + 1) % len(leaves)]]
    if length % 2 == 0:
        e = ["-", e]
    assert len(ops_of_tree(e)) == length
    return e


def _leaves(rng, cols, n_lit_every=5):
    out = []
    for i, c in enumerate(cols):
        out.append(c)
        if i % n_lit_every == n_lit_every - 1:
            out.append(EDGE[i % len(EDGE)] if i % 2 else int(rng.integers(0, P)))
    return out


def _const(rng):
    return EDGE[int(rng.integers(0, len(EDGE)))] if rng.integers(0, 2) else int(rng.integers(0, P))


def rand_tree(rng, cols, size):
    """random tree of about `size` nodes: every operator, constants on either or both sides, unary minus anywhere,
    subtrees made only of constants"""
    if size <= 1:
        return cols[int(rng.integers(0, len(cols)))] if rng.integers(0, 3) else _const(rng)
    kind = int(rng.integers(0, 6))
    if kind == 0:
        return ["-", rand_tree(rng, cols, size - 1)]
    if kind == 1:                                                    # constant-only subtree
        return [_const(rng), "+-*"[int(rng.integers(0, 3))], ["-", _const(rng)] if rng.integers(0, 2) else _const(rng)]
    left = int(rng.integers(1, size))
    return [rand_tree(rng, cols, left), "+-*"[int(rng.integers(0, 3))], rand_tree(rng, cols, size - left)]


def _rand_trees(rng, cols, count, size):
    out = []
    while len(out) < count:
        t = rand_tree(rng, cols, size)
        if stack_depth(ops_of_tree(t)) <= STACK:
            out.append(t)
    return out


def depth_tree(depth, first=0, ops="+-*"):
    """right-leaning tree with stack depth exactly `depth`: pushes c_first .. c_{first+depth-1} (some as literals), then folds"""
    leaves = [x(first + i) if i % 4 != 2 else EDGE[i % len(EDGE)] for i in range(depth)]
    e = leaves[-1]
    for i in range(depth - 2, -1, -1):
        e = [leaves[i], ops[i % len(ops)], e]
    assert stack_depth(ops_of_tree(e)) == depth
    return e


def _w(*items):
    """raw words: ints are opcodes/operands as given; ('x', c) = PUSH_APC c, ('k', v) = PUSH_CONST v"""
    out = []
    for it in items:
        if isinstance(it, tuple):
            out += [M.OP_PUSH_APC if it[0] == "x" else M.OP_PUSH_CONST, it[1]]
        else:
            out.append(it)
    return out


ADD, SUB, MUL, NEG, INV = M.OP_ADD, M.OP_SUB, M.OP_MUL, M.OP_NEG, M.OP_INV_OR_ZERO

INV_RAW = [
    _w(("x", 20), INV),                                          # inv of a column: zero rows give 0
    _w(("k", 0), INV),                                           # inv(0) folded on the host
    _w(("k", 3), INV, INV),                                      # inv(inv(3)) folded
    _w(("x", 21), INV, INV),                                     # inv(inv(x)) = x
    _w(("x", 22), ("x", 22), INV, MUL),                          # is-nonzero: x * inv(x)
    _w(("k", 3), ("k", 3), SUB, INV, ("x", 23), MUL),            # inv of a folded 0, times a column
    _w(("k", P - 1), INV, ("x", 24), ADD),                       # inv(P-1) = P-1
    _w(("x", 25), NEG, INV, ("k", 7), INV, MUL),                 # inv(-x) * inv(7)
    _w(("x", 26), ("k", 1), SUB, INV, ("x", 26), MUL),           # x * inv(x - 1)
    _w(("k", 2), ("k", 5), MUL, INV, ("k", 10), MUL),            # inv(10) * 10 folded to 1
]


def literals_case(seed=1):
    rng = np.random.default_rng(seed)
    H = (P - 1) // 2
    cons = [
        [x(0), "*", 5],                                          # literal on the right of *
        [7, "*", x(1)],                                          # literal on the left
        [[3, "-", 5], "*", x(2)],                                # folded 3 - 5 = P - 2
        [x(3), "*", [["-", 4], "+", 4]],                         # folded -4 + 4 = 0: Shoup product by 0
        [[0, "*", 9], "+", x(4)],                                # product folding to 0
        [["-", 0], "+", 1],                                      # -0 + 1: a constraint that folds to the literal 1
        12345,                                                   # a lone literal
        P - 1,
        x(5),                                                    # a lone column
        [x(6), "*", x(6)],
        [x(7), "-", x(7)],
        [[x(8), "+", x(8)], "*", [x(8), "-", [P - 1, "*", x(8)]]],   # one column read four times
        ["-", [x(9), "*", [x(10), "+", P - 1]]],                 # unary minus over a subtree
        [[P - 1, "*", P - 1], "*", x(11)],                       # folds to 1
        [[H + 1, "*", 2], "-", x(12)],                           # (P+1)/2 * 2 = 1
        [[1 << 27, "*", 15], "+", x(13)],                        # 15 * 2^27 = P - 1
        [[P - 2, "+", 2], "*", [x(14), "*", x(15)]],             # folds to 0 times a product
        [[x(16), "*", [H, "-", H]], "+", [2, "*", [3, "*", [P - 1, "*", 0]]]],
        [["-", [5, "-", 2]], "*", ["-", x(17)]],
        [[H, "+", H], "-", [x(18), "*", [1, "-", 1]]],           # both sides constant after folding: P - 1 - 0
        [["-", [P - 1, "*", 2]], "*", [x(19), "+", [H + 1, "*", [2, "-", 1]]]],
        depth_tree(16, 27),                                      # stack depth exactly 16
        _chain([x(i) for i in range(40)], 2 * 40 - 1),           # 40 distinct columns in one constraint
        _chain(_leaves(rng, [x(i) for i in range(3, 43)]), 101),
    ] + _rand_trees(rng, [x(i) for i in range(48)], 24, 12)
    return Case("literals", 48, cons, INV_RAW)


def modules_case(seed=2):
    """>= 3 JIT modules over 640 columns: a group of exactly 600 ops, a one-constraint group of 601, a module of exactly 2000 words, one
    constraint of 2001 words (a module of its own), and a tail of small constraints"""
    rng = np.random.default_rng(seed)
    W = 640
    cols = [x(i) for i in range(W)]
    few = _leaves(rng, cols[:16])                            # 16 columns: the group cut is by ops alone
    lv = _leaves(rng, cols)
    cons = [_chain(few, 300), _chain(few[3:], 300),          # module 0 (2000 words): a group of exactly 600 ops,
            _chain(few[5:], 300), _chain(few[7:], 301),      # then 300 + 301 = 601 ops, cut into two groups
            _chain(lv, 799)]                                 # 799 ops over > 32 columns: hoisted loads, then __ldg at use
    cons += [_chain(lv[100:], 2001)]                         # module 1: one constraint past the module size
    cons += [_chain(lv[300:], 1000), _chain(lv[50:], 601), _chain(few, 398), x(W - 1)]      # module 2: exactly 2000 words
    cons += _rand_trees(rng, cols, 60, 14)                   # module 3
    return Case("modules", W, cons, [])


def module_bounds(case):
    """constraint indices where air_jit.cuh starts a module (packed words per module <= 2000 unless one constraint is longer)"""
    lens = [len(o) for o in case.constraint_ops()]
    bounds, w = [0], 0
    for k, n in enumerate(lens):
        if w > 0 and w + n > MODULE_WORDS:
            bounds.append(k)
            w = 0
        w += n
    return bounds + [len(lens)]


# ---- interactions: chunk templates (each starts a new chunk after any of the others, see chunk_starts) ----
def _lin(rng, cols):
    c = cols[int(rng.integers(0, len(cols)))]
    k = int(rng.integers(0, 5))
    return [c, "+", _const(rng)] if k == 0 else [[_const(rng), "*", _const(rng)], "*", c] if k == 1 else ["-", c] if k == 2 else c


def _lit_arg(rng):
    k = int(rng.integers(0, 3))
    return _const(rng) if k == 0 else [_const(rng), "-", [_const(rng), "*", _const(rng)]] if k == 1 else ["-", _const(rng)]


MULTS_0 = [0, 1, P - 1, [3, "-", 3], [[P - 1, "*", P - 1], "+", 5]]          # literal and constant-folded multiplicities


def _mult(rng, cols, deg):
    if deg == 0:
        return MULTS_0[int(rng.integers(0, len(MULTS_0)))]
    c = [cols[int(rng.integers(0, len(cols)))] for _ in range(deg)]
    e = c[0] if rng.integers(0, 2) else ["-", c[0]]
    for t in c[1:]:
        e = [e, "*", [t, "+", _const(rng)] if rng.integers(0, 2) else t]
    return e


def _args(rng, cols, n, dyn, quad=False):
    """n arguments; `dyn` of them linear in the columns (or one quadratic), the rest literals / constant subtrees"""
    args = [_lit_arg(rng) for _ in range(n)]
    pos = list(rng.permutation(n)[:dyn]) if n else []
    for p in pos:
        args[p] = _lin(rng, cols)
    if quad and n:
        args[pos[0] if pos else 0] = [cols[0], "*", _lin(rng, cols)]
    return args


def _bus_id(rng):
    return [0, P - 1, 3, 6, 7, 1, 2, int(rng.integers(0, P))][int(rng.integers(0, 8))]


def chunk_template(rng, cols, kind, k=3):
    """kind: 'quad' one interaction with a degree-2 argument; 'pair' two interactions with linear arguments; 'cubic' one linear
    interaction whose multiplicity has degree 3; 'const' k interactions with constant (or no) arguments, the first with a
    degree-3 multiplicity"""
    if kind == "quad":
        return [{"id": _bus_id(rng), "mult": _mult(rng, cols, int(rng.integers(0, 2))), "args": _args(rng, cols, int(rng.integers(1, 12)), 1, quad=True)}]
    if kind == "pair":
        return [{"id": _bus_id(rng), "mult": _mult(rng, cols, int(rng.integers(0, 3)) if i == 0 else int(rng.integers(0, 2))),
                 "args": _args(rng, cols, n, max(1, min(n, int(rng.integers(1, 4)))))}
                for i, n in enumerate(rng.integers(1, 12, size=2))]
    if kind == "cubic":
        return [{"id": _bus_id(rng), "mult": _mult(rng, cols, 3), "args": _args(rng, cols, int(rng.integers(1, 11)), 1)}]
    out = []
    for i in range(k):
        n = [0, 1, 2, 11][int(rng.integers(0, 4))]
        out.append({"id": _bus_id(rng), "mult": _mult(rng, cols, 3 if i == 0 else int(rng.integers(0, 4))), "args": _args(rng, cols, n, 0)})
    return out


def bus_case(name, plan, width=24, seed=0, constraints=()):
    """plan: list of template kinds, or ('const', k); the chunk count is len(plan), checked against chunk_starts"""
    rng = np.random.default_rng(seed)
    cols = [x(i) for i in range(width)]
    bus = []
    for p in plan:
        kind, k = p if isinstance(p, tuple) else (p, 3)
        bus += chunk_template(rng, cols, kind, k)
    cs = chunk_starts(bus)
    assert cs is not None and len(cs) - 1 == len(plan), (name, cs)
    return Case(name, width, constraints, [], bus)


def _plan(n, seed):
    """n chunk templates, never two 'const' in a row (they would merge)"""
    rng = np.random.default_rng(seed)
    kinds, out = ["quad", "pair", "cubic", "const"], []
    for i in range(n):
        k = kinds[int(rng.integers(0, 4))]
        if k == "const" and out and out[-1][0] == "const":
            k = "pair"
        out.append(("const", int(rng.integers(3, 9))) if k == "const" else (k, 0))
    return out


def bus_cases():
    """chunk counts 1, 2, 3, 15, 16, 17 and 35: odd permutation-group tails, module cuts (16 chunks per module), literal arguments and
    multiplicities in every module, constant chunks of 3 to 40 interactions"""
    cases = [
        bus_case("bus_1", [("const", 40)], seed=11),
        bus_case("bus_2", [("pair", 0), ("quad", 0)], seed=12),
        bus_case("bus_3", [("cubic", 0), ("const", 5), ("pair", 0)], seed=13),
    ]
    for n in (15, 16, 17):
        cases.append(bus_case("bus_%d" % n, _plan(n, n), seed=n))
    big = _plan(35, 35)
    big[0], big[17], big[34] = ("const", 3), ("const", 40), ("const", 17)
    if big[1][0] == "const":
        big[1] = ("pair", 0)
    for i in (16, 18, 33):
        if big[i][0] == "const":
            big[i] = ("quad", 0)
    cases.append(bus_case("bus_35", big, width=30, seed=35))
    return cases


def guarded(case, guard=0):
    """the same constraints multiplied by column `guard`: a trace whose guard column is 0 satisfies all of them"""
    cons = [[c, "*", x(guard)] for c in case.constraints]              # guard on the right: the stack depth stays <= 16
    raw = [w + _w(("x", guard), MUL) for w in case.raw]
    return cons, raw


# ---- refusals ----
def refusal_cases():
    """(name, constraints bytecode+spans or None, bus program, expected code): refused by pb_air_compile / pb_air_set_interactions"""
    cols = [x(i) for i in range(20)]
    ok = {"id": 1, "mult": x(0), "args": [x(1)]}
    deg4 = [[x(0), "*", x(1)], "*", [x(2), "*", x(3)]]
    out = []

    def bus(ints):
        m = M.SymbolicMachine([], ints + [{"id": 0, "mult": 0, "args": cols}])
        return M.compile_bus(m, 1)

    out.append(("constraint_depth_17", [depth_tree(17)], None, -3))
    out.append(("mult_degree_4", [], bus([ok, {"id": 2, "mult": deg4, "args": [5]}]), -2))
    out.append(("arg_degree_4", [], bus([{"id": 2, "mult": 1, "args": [3, deg4]}, ok]), -2))
    out.append(("interaction_depth_17", [], bus([ok, {"id": 2, "mult": x(4), "args": [depth_tree(17, ops="+-")]}]), -3))      # linear: refused for its depth alone
    ints, spans, bc = bus([ok, {"id": 2, "mult": x(4), "args": [x(5), 9]}])
    off = len(bc)
    bc = bc + _w(("x", 5), INV)                                   # argument 0 of interaction 1 := inv(c5)
    spans = list(spans)
    spans[ints[1][2] + 1] = (off, 3)
    out.append(("interaction_inv", [], (ints, spans, bc), -2))
    return out


def all_air_cases():
    return [literals_case(), modules_case()]


# ---------------------------------------------------------------- traces
def edge_matrix(width, n, seed):
    """columns of 0, 1, P-1, P-2, alternating 0 / P-1, and random; every fourth row all zero (inv of 0)"""
    rng = np.random.default_rng(seed)
    pats = [lambda: np.zeros(n), lambda: np.ones(n), lambda: np.full(n, P - 1), lambda: np.full(n, P - 2),
            lambda: np.where(np.arange(n) % 2, P - 1, 0), lambda: rng.choice(np.array(EDGE), n), lambda: rng.integers(0, P, n)]
    m = np.stack([pats[(c * 5 + seed) % len(pats)]() for c in range(width)]).astype(np.uint32)
    m[:, ::4] = 0
    return m


def rand_matrix(width, n, seed):
    return np.random.default_rng(seed).integers(0, P, size=(width, n), dtype=np.uint32)
