"""Every Poseidon2 kernel against the plain big-integer reference (tests/py_poseidon2.py) and the C oracle under the same
instantiation, on states and leaf rows chosen round by round (tests/p2_edges.py) so that the S-box, diagonal and external-layer
shortcuts of powdr_b200/csrc/poseidon2.cuh meet their edge words, under four instantiations (p2_edges.instances): Plonky3's (the
add-chain diagonal), random constants with zero round constants and a generic diagonal holding 0, 1, p - 1, 2, (p + 1) / 2, Plonky3's
diagonal with lane 15 changed (generic diagonal), Plonky3's diagonal with other round constants (add-chain diagonal).

What each test reaches:
  * permute_states_kernel (one thread per state, 256-thread CTAs, last CTA partial) and permute_states_coop_kernel (16 lanes per
    state; n = 1, 3, 17 leave a live group beside a dead one in the last warp);
  * pb_merkle_commit at 2^10 rows (leaf_hash_cols_coop_kernel, LEAF_COOP side) and 2^11 rows (leaf_hash_cols_kernel, 128 threads),
    every last-block remainder 0-7 with 0-4 full blocks; above them compress_block_kernel kb = 1 at 2^11, then compress_coop_kernel;
  * pb_merkle_commit_rows8 at 2^10 (leaf_hash_rows8_coop_kernel) and 2^11 (leaf_hash_rows8_kernel);
  * merkle_upper at every height 2^0-2^16 (compress_coop_kernel kb 0-7, compress_block_kernel kb 1-6 at 32-256 threads), 2^19
    (kb = 9, 256 threads), 2^20 and 2^21 (kb = 10: 512 parents on 256 threads, each thread walks the first level twice);
  * whole proofs (leaf, compress, inject, rows8, FRI-challenge and grind kernels with the host transcript) under a generic diagonal;
  * a context whose device constants a later pb_ctx_create put back to the default.
Outputs are compared as the device words the kernels wrote, not after a conversion that would reduce them: a modular add that leaves
p where it should give 0 is harmless inside the permutation and shows only in a word it outputs."""
import contextlib

import numpy as np
import pytest

import p2_edges as E
import py_poseidon2 as pp
from py_poseidon2 import P
from util import rand_field

pytestmark = pytest.mark.gpu

INSTANCES = E.instances()
NAMES = list(INSTANCES)
_EDGES = {}


def edges(name):
    if name not in _EDGES:
        _EDGES[name] = E.edge_states(INSTANCES[name])
    return _EDGES[name]


@pytest.fixture(scope="module")
def pctx():
    """a context of its own: its host transcript constants change with the instantiation, the session's do not"""
    import powdr_b200
    c = powdr_b200.Context(0)
    c.set_fri_params(8, 4)
    yield c
    c.close()


@contextlib.contextmanager
def instantiation(ctx, orc, name):
    """the device bank, ctx's transcript and the oracle under one instantiation; the default back afterwards, whatever happens"""
    inst = INSTANCES[name]
    try:
        ctx.set_poseidon2(*E.as_arrays(inst))
        orc.set_poseidon2(*E.as_arrays(inst))
        yield inst
    finally:
        orc.reset_poseidon2()
        ctx.set_poseidon2(*E.as_arrays(pp.DEFAULT))


def _mont(a):
    """canonical -> the device words a kernel must write (canonical Montgomery form)"""
    return ((np.asarray(a, dtype=np.uint64) * np.uint64(pp.R)) % np.uint64(P)).astype(np.uint32)


def _bad_rows(raw, exp):
    """indices of the rows whose device words differ from the canonical Montgomery form of `exp`"""
    return np.nonzero((raw != _mont(exp)).any(axis=1))[0]


def _expected(orc, inst, states, reps=1):
    out = np.array(states, dtype=np.uint32)
    for _ in range(reps):
        out = np.stack([orc.poseidon2_permute(s) for s in out])
    return out


# ---------------------------------------------------------------- the permutation itself
@pytest.mark.parametrize("reps", [1, 3])
@pytest.mark.parametrize("name", NAMES)
def test_permute_states_on_edge_states(pctx, orc, name, reps):
    es = edges(name)
    st = np.array([e.state for e in es], dtype=np.uint32)          # 362 states: the second CTA is partial
    with instantiation(pctx, orc, name) as inst:
        d = pctx.to_device(st)
        pctx.poseidon2_permute(d.ptr, len(es), reps)
        raw = pctx.to_host(d, st.shape, monty=False)
        exp = _expected(orc, inst, st, reps)
    if reps == 1:
        assert exp.tolist() == [pp.permute(e.state, inst) for e in es]
    bad = [es[i].name for i in _bad_rows(raw, exp)]
    assert not bad, bad[:10]


@pytest.mark.parametrize("n", [1, 3, 17, 1000])
@pytest.mark.parametrize("name", NAMES)
def test_permute_coop_on_edge_states(pctx, orc, name, n):
    es = edges(name)
    idx = [(i * 7) % len(es) for i in range(n)] if n < len(es) else [i % len(es) for i in range(n)]
    st = np.array([es[i].state for i in idx], dtype=np.uint32)
    with instantiation(pctx, orc, name) as inst:
        d = pctx.to_device(st)
        pctx.poseidon2_permute_coop(d.ptr, n)
        raw = pctx.to_host(d, st.shape, monty=False)
        exp = _expected(orc, inst, st)
    bad = [es[idx[i]].name for i in _bad_rows(raw, exp)]
    assert not bad, bad[:10]


# ---------------------------------------------------------------- leaves and trees
def _targeted_matrix(inst, width, log_h, seed):
    """(width, 2^log_h) column-major rows: every targeted leaf row of p2_edges.rows, each followed by a constant-0 and a
    constant-(p - 1) row, spread over the height; random rows elsewhere -> (matrix, positions of the targeted rows, their rows)"""
    h = 1 << log_h
    rng = np.random.default_rng(seed)
    full = rand_field(rng, (h, width))
    targeted = [e.row for e in E.rows(inst, width, seed)]
    stride = h // (3 * len(targeted))
    pos = []
    for k, row in enumerate(targeted):
        at = 3 * k * stride if k + 1 < len(targeted) else h - 3       # the last one at the end of the last CTA
        full[at], full[at + 1], full[at + 2] = row, [0] * width, [P - 1] * width
        pos.append(at)
    return np.ascontiguousarray(full.T), pos, targeted


def _split(width):
    """1-3 matrices whose widths add up to `width`"""
    k = min(width, 1 + width % 3)
    cuts = [width * i // k for i in range(k + 1)]
    return [cuts[i + 1] - cuts[i] for i in range(k)]


def _commit(ctx, mats, log_h):
    """pb_merkle_commit -> (the layer array's device words, root)"""
    h = 1 << log_h
    d_mats = [ctx.to_device(m) for m in mats]
    d_layers = ctx.alloc(32 * 2 * h)
    root = ctx.merkle_commit([d.ptr for d in d_mats], [m.shape[0] for m in mats], log_h, d_layers.ptr)
    return ctx.to_host(d_layers, (2 * h - 1, 8), monty=False), root


def _python_tree_root(leaves, inst):
    level = [list(map(int, x)) for x in leaves]
    while len(level) > 1:
        level = [pp.compress(level[2 * i], level[2 * i + 1], inst) for i in range(len(level) // 2)]
    return level[0]


WIDTHS = list(range(1, 18)) + [24, 25, 31, 32, 33]


@pytest.mark.parametrize("log_h", [10, 11])
@pytest.mark.parametrize("name", NAMES)
def test_merkle_commit_targeted_rows(pctx, orc, name, log_h):
    """both leaf forms at every last-block remainder 0-7 with 0-4 full blocks, split over 1-3 matrices: the whole layer array
    against the oracle, the targeted rows' leaves against the reference, one root against the reference over the leaves"""
    with instantiation(pctx, orc, name) as inst:
        for w in WIDTHS:
            full, pos, targeted = _targeted_matrix(inst, w, log_h, seed=w)
            widths = _split(w)
            mats = [np.ascontiguousarray(full[sum(widths[:i]):sum(widths[:i + 1])]) for i in range(len(widths))]
            raw, root = _commit(pctx, mats, log_h)
            exp = np.concatenate(orc.merkle_commit(mats))
            bad = _bad_rows(raw, exp)
            assert bad.size == 0, (w, widths, bad[:10].tolist())
            assert root == exp[-1].tolist()
            for at, row in zip(pos, targeted):
                assert exp[at].tolist() == pp.hash_row(row, inst), (w, at)
            if w == 9:
                assert _python_tree_root(exp[:1 << log_h], inst) == root


@pytest.mark.parametrize("log_h", [10, 11])
@pytest.mark.parametrize("name", NAMES)
def test_merkle_commit_rows8_targeted_rows(pctx, orc, name, log_h):
    with instantiation(pctx, orc, name) as inst:
        full, pos, targeted = _targeted_matrix(inst, 8, log_h, seed=log_h)
        rows = np.ascontiguousarray(full.T)                            # row-major [h][8]
        h = 1 << log_h
        d = pctx.to_device(rows)
        d_layers = pctx.alloc(32 * 2 * h)
        root = pctx.merkle_commit_rows8(d.ptr, log_h, d_layers.ptr)
        raw = pctx.to_host(d_layers, (2 * h - 1, 8), monty=False)
        exp = np.concatenate(orc.merkle_commit([full]))
        bad = _bad_rows(raw, exp)
        assert bad.size == 0, bad[:10].tolist()
        assert root == exp[-1].tolist()
        for at, row in zip(pos, targeted):
            assert exp[at].tolist() == pp.hash_row(row, inst), at


@pytest.mark.parametrize("name", ["plonky3", "random_zero_rc"])
def test_merkle_upper_every_height(pctx, orc, name):
    """every launch shape of merkle_upper up to 2^16 leaves: the whole layer array against the oracle"""
    with instantiation(pctx, orc, name):
        for log_h in range(17):
            rng = np.random.default_rng(log_h)
            mats = [rand_field(rng, (3, 1 << log_h))]
            raw, _ = _commit(pctx, mats, log_h)
            exp = np.concatenate(orc.merkle_commit(mats))
            bad = _bad_rows(raw, exp)
            assert bad.size == 0, (log_h, bad[:10].tolist())


@pytest.mark.parametrize("log_h", [19, 20, 21])
def test_merkle_upper_tall_trees(ctx, orc, log_h):
    """compress_block_kernel at kb = 9 (2^19 leaves) and kb = 10 (2^20, 2^21: two passes of 256 threads over 512 first-level
    parents): the whole layer array against the AVX-512 oracle (default instantiation)"""
    rng = np.random.default_rng(log_h)
    mats = [rand_field(rng, (1, 1 << log_h))]
    raw, root = _commit(ctx, mats, log_h)
    exp = np.concatenate(orc.fast_merkle_commit(mats))
    bad = _bad_rows(raw, exp)
    assert bad.size == 0, bad[:10].tolist()
    assert root == exp[-1].tolist()


# ---------------------------------------------------------------- whole proofs under another instantiation
# heights 2 to 2^11 with interactions: both leaf forms, injection of the shorter heights, both compress forms, rows8 FRI layers,
# the device FRI challenges and the proof of work.  Chips with constraints have all-zero traces, which satisfy them.
PROOF_SPEC = [(11, 6, 0, 4), (10, 5, 0, 3), (6, 7, 2, 0, True), (3, 4, 0, 2), (1, 5, 0, 2)]


def _prove_all(ctx, chips, on_device):
    airs = [ctx.air(bc, spans, t.shape[0], bus) for t, bc, spans, bus in chips]
    if on_device:
        bufs = [ctx.to_device(t) for t, _, _, _ in chips]
        ptrs = [b.ptr for b in bufs]
    else:
        bufs = [((t.astype(np.uint64) * np.uint64((1 << 32) % P)) % np.uint64(P)).astype(np.uint32) for t, _, _, _ in chips]
        ptrs = [b.ctypes.data for b in bufs]
    out = ctx.prove_chips([(a, p, t.shape[1].bit_length() - 1, t.shape[0]) for a, p, (t, _, _, _) in zip(airs, ptrs, chips)],
                          on_device=on_device)
    for a in airs:
        a.free()
    return out


def _keys(chips):
    from powdr_b200 import VerifyingKey
    return [(VerifyingKey(bc, sp, t.shape[0], bus), t.shape[1].bit_length() - 1) for t, bc, sp, bus in chips]


@pytest.mark.parametrize("name", ["random_zero_rc", "p3_diag_lane15"])
def test_proofs_under_another_instantiation(pctx, orc, name):
    from powdr_b200 import verify_chips, verify_segment
    from powdr_b200.capi import PB_ERR_REJECTED
    from test_gpu_chips import _chips
    chips = _chips(PROOF_SPEC, seed=9)
    seg = _chips([(11, 8, 0, 5)], seed=10)
    before = _prove_all(pctx, chips, True)
    consts = E.as_arrays(INSTANCES[name])
    with instantiation(pctx, orc, name):
        exp = orc.prove_chips(chips, n_queries=8, pow_bits=4)
        for on_device in (True, False):
            proof, cs, ys, q = _prove_all(pctx, chips, on_device)
            assert proof == exp[0] and (cs == exp[1]).all() and (ys == exp[2]).all() and (q == exp[3]).all(), on_device
        assert orc.verify_chips(chips, proof, cs, ys, q) == 0
        keys = _keys(chips)
        assert verify_chips(keys, proof, cs, ys, q, n_queries=8, pow_bits=4, poseidon2=consts) == (0, 0)
        assert verify_chips(keys, proof, cs, ys, q, n_queries=8, pow_bits=4)[0] == PB_ERR_REJECTED
        # the single-chip prover
        (trace, bc, spans, bus), = seg
        air = pctx.air(bc, spans, trace.shape[0], bus)
        d = pctx.to_device(trace)
        sproof = pctx.prove_segment(air, d.ptr, 11, trace.shape[0], on_device=True)
        sq, sys_ = pctx.query_segment(11, trace.shape[0], air.perm_width)
        air.free()
        e_s, e_ys, e_q, _ = orc.prove(trace, bc, spans, bus, n_queries=8, pow_bits=4)
        assert sproof == e_s and (sys_ == e_ys).all() and (sq == e_q).all()
        (vk, log_n), = _keys(seg)
        assert verify_segment(vk, log_n, sproof, sys_, sq, n_queries=8, pow_bits=4, poseidon2=consts) == (0, 0)
        assert verify_segment(vk, log_n, sproof, sys_, sq, n_queries=8, pow_bits=4)[0] == PB_ERR_REJECTED
    after = _prove_all(pctx, chips, True)
    assert before[0] == after[0] and all((a == b).all() for a, b in zip(before[1:], after[1:]))
    assert before[0] != proof


def test_a_later_context_resets_the_device_constants(pctx, orc):
    """pb_ctx_create uploads the default constants to the GPU's one constant bank, so a context that set others then hashes on the
    device with the default while its transcript replays the custom ones: the device-sampled FRI challenges disagree with the host
    replay and the proof ends in PB_ERR_INTERNAL instead of returning a proof"""
    import powdr_b200
    from powdr_b200.capi import PB_ERR_INTERNAL, PbError
    from test_gpu_chips import _chips
    chips = _chips(PROOF_SPEC[:2], seed=4)
    with instantiation(pctx, orc, "random_zero_rc"):
        other = powdr_b200.Context(0)
        other.close()
        with pytest.raises(PbError) as err:
            _prove_all(pctx, chips, True)
        assert err.value.code == PB_ERR_INTERNAL
    proof, cs, ys, q = _prove_all(pctx, chips, True)            # defaults on both sides again
    exp = orc.prove_chips(chips, n_queries=8, pow_bits=4)
    assert proof == exp[0] and (q == exp[3]).all()
