"""A second, independent restatement of Poseidon2 (width 16, x^7, 4+13+4 rounds) in pure Python big-integer arithmetic, written
from the Poseidon2 paper's round structure and driven only by constants/poseidon2_babybear_w16.json -- it shares no code with
oracle/poseidon2.c.  tests/test_oracle.py checks the C oracle against it (permutation, sponge, compression, a Merkle root).

The instantiation is data (`Instance`: round constants and internal diagonal, canonical); every function takes one and defaults to
the JSON constants.  The permutation is invertible round by round (`inverse`, `entry_to_input`), and `trace` records what each round
sees as the kernels hold it: the Montgomery word c * 2^32 mod p of every value."""
import json
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K = json.load(open(os.path.join(ROOT, "constants", "poseidon2_babybear_w16.json")))
P = K["p"]
R = (1 << 32) % P
R_INV = pow(R, -1, P)
D_INV = pow(7, -1, P - 1)        # x -> x^D_INV undoes the S-box x -> x^7 (gcd(7, p - 1) = 1)
N_ROUNDS = 21                    # rounds 0-3 external, 4-16 internal, 17-20 external


def mont(c):
    """the device word of canonical c"""
    return c * R % P


def unmont(w):
    """the canonical value of device word w"""
    return w * R_INV % P


class Instance:
    """rc_ext [8][16] (rounds 0-3, then 17-20), rc_int [13], diag [16] (internal matrix 1 + diag(V)), canonical"""

    def __init__(self, rc_ext, rc_int, diag):
        self.rc_ext = [[int(x) % P for x in row] for row in rc_ext]
        self.rc_int = [int(x) % P for x in rc_int]
        self.diag = [int(x) % P for x in diag]
        assert len(self.rc_ext) == 8 and all(len(r) == 16 for r in self.rc_ext) and len(self.rc_int) == 13 and len(self.diag) == 16
        self._int_inv = None

    def round_rc(self, r):
        """round r's constants: a list of 16 for an external round, one value for an internal one"""
        if r < 4:
            return self.rc_ext[r]
        if r < 17:
            return self.rc_int[r - 4]
        return self.rc_ext[r - 13]

    def internal_inverse(self):
        if self._int_inv is None:
            self._int_inv = mat_inverse([[(1 + (self.diag[i] if i == j else 0)) % P for j in range(16)] for i in range(16)])
        return self._int_inv


DEFAULT = Instance(K["external_initial"] + K["external_terminal"], K["internal"], K["internal_diag_m1"])


def is_external(r):
    return r < 4 or r >= 17


def external(s):
    """circ(2 M4, M4, M4, M4): every 4-chunk is multiplied by M4, then the sum of the four chunks is added to each"""
    m4 = K["m4"]
    chunks = [[sum(m4[i][j] * s[4 * c + j] for j in range(4)) % P for i in range(4)] for c in range(4)]
    tot = [sum(chunks[c][i] for c in range(4)) % P for i in range(4)]
    return [(chunks[c][i] + tot[i]) % P for c in range(4) for i in range(4)]


def internal(s, inst=DEFAULT):
    """(J + diag(V)): y_i = V_i x_i + sum(x)"""
    tot = sum(s) % P
    return [(inst.diag[i] * s[i] + tot) % P for i in range(16)]


def sbox_layer(s, r, inst=DEFAULT):
    """round r's constant addition and S-box (all lanes of an external round, lane 0 of an internal one)"""
    rc = inst.round_rc(r)
    if is_external(r):
        return [pow((x + c) % P, 7, P) for x, c in zip(s, rc)]
    return [pow((s[0] + rc) % P, 7, P)] + list(s[1:])


def sbox_layer_inv(s, r, inst=DEFAULT):
    rc = inst.round_rc(r)
    if is_external(r):
        return [(pow(x, D_INV, P) - c) % P for x, c in zip(s, rc)]
    return [(pow(s[0], D_INV, P) - rc) % P] + list(s[1:])


def linear_layer(s, r, inst=DEFAULT):
    return external(s) if is_external(r) else internal(s, inst)


def mat_vec(m, v):
    return [sum(a * b for a, b in zip(row, v)) % P for row in m]


def mat_inverse(m):
    """Gauss-Jordan mod p; raises ValueError on a singular matrix"""
    n = len(m)
    a = [[int(x) % P for x in row] + [1 if i == j else 0 for j in range(n)] for i, row in enumerate(m)]
    for c in range(n):
        piv = next((i for i in range(c, n) if a[i][c]), None)
        if piv is None:
            raise ValueError("singular matrix")
        a[c], a[piv] = a[piv], a[c]
        inv = pow(a[c][c], -1, P)
        a[c] = [x * inv % P for x in a[c]]
        for i in range(n):
            if i != c and a[i][c]:
                f = a[i][c]
                a[i] = [(x - f * y) % P for x, y in zip(a[i], a[c])]
    return [row[n:] for row in a]


EXT_MATRIX = [list(col) for col in zip(*[external([1 if i == j else 0 for i in range(16)]) for j in range(16)])]
EXT_INV = mat_inverse(EXT_MATRIX)


def permute(state, inst=DEFAULT):
    s = [int(x) % P for x in state]
    assert len(s) == 16
    s = external(s)
    for r in range(N_ROUNDS):
        s = linear_layer(sbox_layer(s, r, inst), r, inst)
    return s


def trace(state, inst=DEFAULT):
    """the forward pass as the kernels see it, in device words: {("entry", r): state entering round r (its S-box inputs before the
    constant), ("lin", r): input of round r's linear layer, ("lin", -1): input of the initial external layer, ("exit", 20): the
    output}; "out": the output, canonical"""
    s = [int(x) % P for x in state]
    t = {("lin", -1): [mont(x) for x in s]}
    s = external(s)
    for r in range(N_ROUNDS):
        t[("entry", r)] = [mont(x) for x in s]
        s = sbox_layer(s, r, inst)
        t[("lin", r)] = [mont(x) for x in s]
        s = linear_layer(s, r, inst)
    t[("exit", N_ROUNDS - 1)] = [mont(x) for x in s]
    t["out"] = s
    return t


def entry_to_input(s, r, inst=DEFAULT):
    """the permutation input whose state entering round r is s (canonical)"""
    s = [int(x) % P for x in s]
    for q in range(r - 1, -1, -1):
        s = mat_vec(EXT_INV if is_external(q) else inst.internal_inverse(), s)
        s = sbox_layer_inv(s, q, inst)
    return mat_vec(EXT_INV, s)


def inverse(state, inst=DEFAULT):
    s = [int(x) % P for x in state]
    for q in range(N_ROUNDS - 1, -1, -1):
        s = mat_vec(EXT_INV if is_external(q) else inst.internal_inverse(), s)
        s = sbox_layer_inv(s, q, inst)
    return mat_vec(EXT_INV, s)


def hash_row(row, inst=DEFAULT):
    """PaddingFreeSponge<16, 8, 8>: overwrite-mode absorption of 8 elements at a time, permute after every (partial) block"""
    s = [0] * 16
    row = [int(x) for x in row]
    for i in range(0, len(row), 8):
        blk = row[i:i + 8]
        s[:len(blk)] = blk
        s = permute(s, inst)
    return s[:8]


def compress(left, right, inst=DEFAULT):
    """TruncatedPermutation<16 -> 8> on left || right"""
    return permute([int(x) for x in left] + [int(x) for x in right], inst)[:8]


def merkle_root(rows, inst=DEFAULT):
    level = [hash_row(r, inst) for r in rows]
    while len(level) > 1:
        level = [compress(level[2 * i], level[2 * i + 1], inst) for i in range(len(level) // 2)]
    return level[0]


class DuplexChallenger:
    """DuplexChallenger<F, Perm16, WIDTH 16, RATE 8> restated from its published behaviour: observing clears pending outputs and
    buffers the value, a full input buffer is absorbed (overwrite) and permuted; sampling absorbs any pending input first and
    pops from the END of the 8-element output buffer."""

    def __init__(self, inst=DEFAULT):
        self.state, self.inp, self.out, self.inst = [0] * 16, [], [], inst

    def _duplex(self):
        self.state[:len(self.inp)] = self.inp
        self.inp = []
        self.state = permute(self.state, self.inst)
        self.out = self.state[:8]

    def observe(self, vals):
        for v in vals:
            self.out = []
            self.inp.append(int(v))
            if len(self.inp) == 8:
                self._duplex()

    def sample(self):
        if self.inp or not self.out:
            self._duplex()
        return self.out.pop()
