"""Poseidon2 states chosen round by round: for each round, the words (Montgomery form, as the kernels hold them) that a state should
carry into that round, walked back to the permutation input through py_poseidon2's inverse.  The word classes are the ones the CUDA
arithmetic takes shortcuts on (powdr_b200/csrc/poseidon2.cuh): the signed S-box argument at 0, +-1 and the ends of [-p, p); the
Plonky3 internal diagonal's div_2k / halve / dbl lanes at their carry and borrow edges; round sums of 0 and p - 1; modular adds in the
external layer that sum to exactly p, also where they make an output word.  A random state reaches any one of these at a chosen place with probability ~2^-31.

Every state carries its claims, (trace key, lane, word), which py_poseidon2.trace must reproduce; `rows` gives leaf rows (8 free
words) whose first S-box layer hits the same classes, by solving the first external layer's 8 x 8 block."""
import random

import py_poseidon2 as pp
from py_poseidon2 import P, mont, unmont

HALF_LO, HALF_HI = (P - 1) // 2, (P + 1) // 2
# S-box classes: the device word s entering the S-box (x = s + (rc_m - p) in [-p, p))
SBOX_WORDS = {"zero": 0, "one": 1, "pm1": P - 1, "pm2": P - 2, "half_lo": HALF_LO, "half_hi": HALF_HI, "2^27": 1 << 27,
              "2^27-1": (1 << 27) - 1}
SBOX_RC = {"arg0": 0, "arg+1": 1, "arg-1": -1}      # s = p - rc_m + d: the argument x is d
SBOX_CLASSES = list(SBOX_WORDS) + list(SBOX_RC)
# internal-layer inputs of the Plonky3 diagonal [-2,1,2,1/2,3,4,-1/2,-3,-4,2^-8,1/4,1/8,2^-27,-2^-8,-1/16,-2^-27]
DIV_LANES = {9: 8, 10: 2, 11: 3, 12: 27, 13: 8, 14: 4, 15: 27}
HALVE_LANES = (3, 6)
DBL_LANES = (2, 4, 5, 7, 8)
DIAG_PATTERNS = ("low0", "low1", "pow2k", "pow2k-1", "p-pow2k")
SUM_CLASSES = {"sum0": 0, "sum_pm1": P - 1}
EXT_PATTERNS = {"all_pm1": [P - 1] * 16, "all_0": [0] * 16, "alt_0_pm1": [0, P - 1] * 8, "alt_1_pm1": [1, P - 1] * 8}
# output lanes that are 0 beside random ones: the last external layer's add sums to exactly p there, and only a canonical result
# tells its reduction apart from one that leaves p (which every later step would still treat as 0)
OUT_ZEROS = {"even": range(0, 16, 2), "odd": range(1, 16, 2), "digest": range(8), "capacity": range(8, 16)}
CLASSES = ["sbox:" + c for c in SBOX_CLASSES] + ["diag:" + d for d in DIAG_PATTERNS] + ["sum:" + s for s in SUM_CLASSES] + \
          ["ext:" + e for e in EXT_PATTERNS] + ["out:" + o for o in OUT_ZEROS]
EXT_LAYERS = [-1, 0, 1, 2, 3, 17, 18, 19, 20]        # the external layers' inputs: the permutation input, then after those rounds


def _rand_u32(rng):
    return rng.randrange(P)


def sbox_word(cls, rc_canon):
    """the device word of S-box class `cls` at a lane whose round constant is rc_canon"""
    if cls in SBOX_WORDS:
        return SBOX_WORDS[cls]
    return (P - mont(rc_canon) + SBOX_RC[cls]) % P


def diag_word(pattern, lane, rng):
    """device word of an internal-layer input lane under a diagonal-edge pattern"""
    if lane in DIV_LANES:
        k = DIV_LANES[lane]
        top = (P - 1) >> k                              # values v << k with v <= top stay below p
        if pattern == "low0":
            return rng.randint(1, top) << k
        if pattern == "low1":
            return (rng.randint(0, top - 1) << k) | ((1 << k) - 1)
        if pattern == "pow2k":
            return 1 << k
        if pattern == "pow2k-1":
            return (1 << k) - 1
        return P - (1 << k)
    if lane in HALVE_LANES:
        return {"low0": 2 * rng.randrange(1, HALF_LO), "low1": 2 * rng.randrange(HALF_LO) + 1, "pow2k": P - 1, "pow2k-1": 1,
                "p-pow2k": P - 2}[pattern]
    if lane in DBL_LANES:
        return {"low0": HALF_HI, "low1": P - 1, "pow2k": P - 2, "pow2k-1": HALF_HI + 1, "p-pow2k": rng.randrange(HALF_HI, P)}[pattern]
    return {"low0": 0, "low1": P - 1, "pow2k": 1, "pow2k-1": HALF_LO, "p-pow2k": HALF_HI}[pattern]


class Edge:
    """name, input state (canonical), claims [(trace key, lane, device word)]; a leaf row's Edge also has the row"""

    def __init__(self, name, state, claims, row=None):
        self.name, self.state, self.claims, self.row = name, state, claims, row

    def reached(self, inst):
        t = pp.trace(self.state, inst)
        return all(t[key][lane] == w for key, lane, w in self.claims)


def _from_entry(name, r, words, inst, claims):
    state = pp.entry_to_input([unmont(w) for w in words], r, inst)
    return Edge(name, state, claims)


def _from_lin(name, r, words, inst):
    """a state whose round-r linear layer sees `words` (r = -1: the input itself)"""
    canon = [unmont(w) for w in words]
    claims = [(("lin", r), i, w) for i, w in enumerate(words)]
    if r < 0:
        return Edge(name, canon, claims)
    return Edge(name, pp.entry_to_input(pp.sbox_layer_inv(canon, r, inst), r, inst), claims)


def edge_states(inst, seed=0):
    """every class at every round it applies to -> [Edge]"""
    rng = random.Random(seed)
    out = []
    for r in range(pp.N_ROUNDS):
        rc = inst.round_rc(r)
        if pp.is_external(r):
            for cls in SBOX_CLASSES:
                words = [sbox_word(cls, rc[i]) for i in range(16)]
                out.append(_from_entry("sbox:%s:r%d" % (cls, r), r, words, inst, [(("entry", r), i, w) for i, w in enumerate(words)]))
            continue
        # internal round: lane 0 takes an S-box class, lanes 1..15 pass to the internal layer untouched and take a diagonal pattern
        for k, cls in enumerate(SBOX_CLASSES):
            pat = DIAG_PATTERNS[k % len(DIAG_PATTERNS)]
            words = [sbox_word(cls, rc)] + [diag_word(pat, i, rng) for i in range(1, 16)]
            claims = [(("entry", r), 0, words[0])] + [(("lin", r), i, words[i]) for i in range(1, 16)]
            out.append(_from_entry("sbox:%s:r%d" % (cls, r), r, words, inst, claims))
        for pat in DIAG_PATTERNS:
            words = [_rand_u32(rng)] + [diag_word(pat, i, rng) for i in range(1, 16)]
            out.append(_from_entry("diag:%s:r%d" % (pat, r), r, words, inst, [(("lin", r), i, words[i]) for i in range(1, 16)]))
        for cls, target in SUM_CLASSES.items():
            lin = [0] + [_rand_u32(rng) for _ in range(15)]
            lin[0] = (target - sum(lin[1:])) % P          # device words add like canonical ones: the round sum is `target`
            out.append(_from_lin("sum:%s:r%d" % (cls, r), r, lin, inst))
    for r in EXT_LAYERS:
        for pat, words in EXT_PATTERNS.items():
            out.append(_from_lin("ext:%s:l%d" % (pat, r), r, list(words), inst))
    for pat, zeros in OUT_ZEROS.items():
        res = [0 if i in zeros else _rand_u32(rng) for i in range(16)]
        out.append(Edge("out:%s:r20" % pat, pp.inverse(res, inst), [(("exit", 20), i, 0) for i in zeros]))
    return out


def class_of(edge_name):
    return edge_name.rsplit(":", 1)[0]


def rows(inst, width, seed=0):
    """leaf rows of `width` words whose first permutation enters round 0 with S-box classes on lanes < min(width, 8), plus rows that
    put the external-layer patterns on the first block -> [Edge] (row: the row; state and claims: its first permutation)"""
    rng = random.Random(seed)
    n = min(width, 8)
    lanes = list(range(n))
    block = None
    while n and block is None:
        try:
            block = pp.mat_inverse([[pp.EXT_MATRIX[i][j] for j in lanes] for i in lanes])
        except ValueError:                               # a singular leading block: target one lane fewer
            n -= 1
            lanes = list(range(n))
    out = []
    for cls in SBOX_CLASSES:
        words = [sbox_word(cls, inst.rc_ext[0][i]) for i in lanes]
        first = pp.mat_vec(block, [unmont(w) for w in words]) if n else []
        row = first + [_rand_u32(rng) for _ in range(width - n)]
        out.append(Edge("sbox:%s:r0" % cls, first_block(row), [(("entry", 0), i, w) for i, w in zip(lanes, words)], row))
    for pat, words in EXT_PATTERNS.items():
        row = [unmont(w) for w in words[:min(width, 8)]] + [_rand_u32(rng) for _ in range(width - min(width, 8))]
        out.append(Edge("ext:%s:l-1" % pat, first_block(row), [(("lin", -1), i, words[i]) for i in range(min(width, 8))], row))
    return out


def first_block(row):
    """the state of a leaf row's first sponge permutation"""
    blk = [int(x) for x in row[:8]]
    return blk + [0] * (16 - len(blk))


def instances(seed=5):
    """the four instantiations the edge tests run under -> {name: Instance}"""
    rng = random.Random(seed)
    d = pp.DEFAULT
    rc_ext = [[rng.randrange(P) for _ in range(16)] for _ in range(8)]
    rc_int = [rng.randrange(P) for _ in range(13)]
    for r, i in ((0, 3), (0, 11), (2, 0), (5, 7), (7, 15)):
        rc_ext[r][i] = 0                                  # a zero constant with s = 0 is the only way to x = -p
    rc_int[0] = rc_int[6] = rc_int[12] = 0
    diag = [rng.randrange(P) for _ in range(16)]
    diag[0], diag[3], diag[6], diag[9], diag[12] = 0, 1, P - 1, 2, HALF_HI
    lane15 = list(d.diag)
    lane15[15] = (lane15[15] + 1) % P                     # only the last entry differs from Plonky3's: the generic diagonal
    rc_ext2 = [[rng.randrange(P) for _ in range(16)] for _ in range(8)]
    rc_int2 = [rng.randrange(P) for _ in range(13)]
    return {
        "plonky3": d,
        "random_zero_rc": pp.Instance(rc_ext, rc_int, diag),
        "p3_diag_lane15": pp.Instance(d.rc_ext, d.rc_int, lane15),
        "p3_diag_other_rc": pp.Instance(rc_ext2, rc_int2, d.diag),
    }


def as_arrays(inst):
    """(rc_ext [8][16], rc_int [13], diag [16]) as uint32 arrays, for pb_ctx_set_poseidon2 / orc.set_poseidon2 / verify params"""
    import numpy as np
    return (np.array(inst.rc_ext, dtype=np.uint32), np.array(inst.rc_int, dtype=np.uint32), np.array(inst.diag, dtype=np.uint32))
