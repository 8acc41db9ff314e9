"""Poseidon2 at the edges its fast arithmetic relies on, without a GPU: the plain big-integer reference (tests/py_poseidon2.py) checks
itself (inverse, known answer, every targeted word reached), then the C oracle, the host transcript's permutation and the AVX-512
Merkle tree are held to it on the states of tests/p2_edges.py, under four instantiations: Plonky3's, random constants with zero round
constants and a generic diagonal holding 0, 1, p - 1, 2 and (p + 1) / 2, Plonky3's diagonal with lane 15 changed, and Plonky3's
diagonal with other round constants."""
import ctypes as C
import functools
import random

import numpy as np
import pytest

import p2_edges as E
import py_poseidon2 as pp
from py_poseidon2 import P

INSTANCES = E.instances()
KAT_OUT = [1906786279, 1737026427, 1959749225, 700325316, 1638050605, 1021608788, 1726691001, 1761127344, 1552405120, 417318995,
           36799261, 1215172152, 614923223, 1300746575, 957311597, 304856115]


@functools.lru_cache(maxsize=None)
def edges(name):
    return E.edge_states(INSTANCES[name])


def by_class(name, cls):
    out = [e for e in edges(name) if E.class_of(e.name) == cls]
    assert out, (name, cls)
    return out


def test_edge_state_counts():
    """every class occurs in the rounds it applies to: 11 S-box classes in all 21 rounds, 5 diagonal patterns and 2 round sums in
    the 13 internal rounds, 4 external patterns at the 9 external layers, 4 output patterns"""
    for name in INSTANCES:
        names = [e.name for e in edges(name)]
        assert len(names) == len(set(names)) == 21 * 11 + 13 * (5 + 2) + 9 * 4 + 4
        assert sorted({E.class_of(n) for n in names}) == sorted(E.CLASSES)


@pytest.mark.parametrize("name", list(INSTANCES))
def test_inverse_undoes_the_permutation(name):
    inst = INSTANCES[name]
    rng = random.Random(3)
    states = [e.state for e in edges(name)[::7]] + [[rng.randrange(P) for _ in range(16)] for _ in range(8)] + [[0] * 16, [P - 1] * 16]
    for s in states:
        assert pp.inverse(pp.permute(s, inst), inst) == s
        assert pp.permute(pp.inverse(s, inst), inst) == s
        assert pp.trace(s, inst)["out"] == pp.permute(s, inst)


def test_reference_known_answer():
    """the committed Plonky3 vector (tests/test_oracle.py::test_poseidon2_plonky3_default_known_answer), forwards and backwards"""
    assert pp.permute(list(range(16))) == KAT_OUT
    assert pp.inverse(KAT_OUT) == list(range(16))


@pytest.mark.parametrize("cls", E.CLASSES)
@pytest.mark.parametrize("name", list(INSTANCES))
def test_edge_states_reach_their_words_and_the_oracle_agrees(orc, name, cls):
    """the instrumented pass reaches every claimed word, and orc.poseidon2_permute_with equals the reference on the state"""
    inst = INSTANCES[name]
    rc_ext, rc_int, diag = E.as_arrays(inst)
    for e in by_class(name, cls):
        t = pp.trace(e.state, inst)
        for key, lane, w in e.claims:
            assert t[key][lane] == w, (e.name, key, lane)
        got = orc.poseidon2_permute_with(np.array(e.state, dtype=np.uint32), rc_ext, rc_int, diag)
        assert got.tolist() == t["out"], e.name


def test_instances_take_the_intended_diagonal_paths():
    """instantiation 3 differs from Plonky3's diagonal in lane 15 only; 4 keeps the diagonal and changes every round constant; 2 has
    zero round constants and the small diagonal entries"""
    d = pp.DEFAULT.diag
    l15 = INSTANCES["p3_diag_lane15"].diag
    assert l15[:15] == d[:15] and l15[15] != d[15]
    o = INSTANCES["p3_diag_other_rc"]
    assert o.diag == d and all(a != b for a, b in zip(o.rc_int, pp.DEFAULT.rc_int))
    r = INSTANCES["random_zero_rc"]
    assert {0, 1, P - 1, 2, (P + 1) // 2} <= set(r.diag) and 0 in r.rc_int and any(0 in row for row in r.rc_ext)


@pytest.mark.parametrize("name", list(INSTANCES))
def test_oracle_runs_under_a_set_instantiation(orc, name):
    """orc.set_poseidon2 switches the oracle's permutation, sponge and compression; reset restores the default"""
    inst = INSTANCES[name]
    rng = random.Random(11)
    orc.set_poseidon2(*E.as_arrays(inst))
    try:
        for e in edges(name)[::5]:
            assert orc.poseidon2_permute(np.array(e.state, dtype=np.uint32)).tolist() == pp.permute(e.state, inst), e.name
        for w in (1, 7, 8, 9, 17, 33):
            for e in E.rows(inst, w)[::3]:
                assert orc.hash_row(np.array(e.row, dtype=np.uint32)).tolist() == pp.hash_row(e.row, inst)
        for _ in range(4):
            l, r = [rng.randrange(P) for _ in range(8)], [rng.randrange(P) for _ in range(8)]
            assert orc.compress(l, r).tolist() == pp.compress(l, r, inst)
    finally:
        orc.reset_poseidon2()
    assert orc.poseidon2_permute(np.arange(16, dtype=np.uint32)).tolist() == KAT_OUT


@pytest.mark.parametrize("cls", E.CLASSES)
def test_host_transcript_permutation_on_edge_states(cls):
    """pb_host_poseidon2_permute (AVX-512 where the CPU has it, and the scalar code) on the default instantiation's edge states"""
    import powdr_b200
    from powdr_b200 import build
    build.build()
    lib = powdr_b200.load_library()
    for e in by_class("plonky3", cls):
        exp = pp.permute(e.state)
        for force_scalar in (0, 1):
            st = (C.c_uint32 * 16)(*e.state)
            assert lib.pb_host_poseidon2_permute(st, 1, force_scalar, None) == 0
            assert list(st) == exp, (e.name, force_scalar)


@pytest.mark.parametrize("widths", [[1], [5], [8], [3, 6], [17], [4, 4, 1], [33]])
def test_fast_merkle_commit_on_targeted_rows(orc, widths):
    """orc.fast_merkle_commit (AVX-512) over rows whose first permutation hits the edge classes, interleaved with constant-0 and
    constant-(p - 1) rows: every leaf and the root against the reference, every layer against the scalar oracle"""
    inst = pp.DEFAULT
    w = sum(widths)
    targeted = [e.row for e in E.rows(inst, w)]
    rows = []
    for r in targeted:
        rows += [r, [0] * w, [P - 1] * w]
    h = 1 << max(4, (len(rows) - 1).bit_length())
    rng = random.Random(w)
    rows += [[rng.randrange(P) for _ in range(w)] for _ in range(h - len(rows))]
    full = np.array(rows, dtype=np.uint32).T
    mats, c0 = [], 0
    for wi in widths:
        mats.append(np.ascontiguousarray(full[c0:c0 + wi]))
        c0 += wi
    got = orc.fast_merkle_commit(mats)
    for i, r in enumerate(rows):
        assert got[0][i].tolist() == pp.hash_row(r, inst), i
    assert got[-1][0].tolist() == pp.merkle_root(rows, inst)
    exp = orc.merkle_commit(mats)
    assert all((a == b).all() for a, b in zip(got, exp))
