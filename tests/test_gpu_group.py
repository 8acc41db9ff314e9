"""All chips of a segment on the ranks of ONE process through the library's group (pb_prove_chips_group / pb_query_chips_group): the
library runs one thread per rank and exchanges device to device.  The group's answer must equal pb_prove_chips + pb_query_chips on the
gathered traces and the oracle's, whatever the world, the FRI switch point or the row sub-blocks; the cross-rank rules are refused before
any rank starts; a rank that fails alone ends the call on every rank."""
import ctypes as C
import os
import subprocess
import threading

import numpy as np
import pytest

from test_gpu_chips import _chips
from test_gpu_sharded_chips import MIXES, _raise, _same, _single
from test_gpu_sharded_row_blocks import SPEC, _shapes

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID = -1


class Ranks:
    """`world` contexts (rank r on devices[r], default 0) with their AIRs and column blocks of `chips`; args[r] as Group.prove_chips
    takes them.  close() frees the groups made by group() first, then the rest."""

    def __init__(self, world, chips, devices=None, fri_params=(8, 4)):
        from powdr_b200.capi import Context
        from powdr_b200.sharded import shard_columns
        self.world, self.ctxs, self.airs, self.bufs, self.args, self.groups = world, [], [], [], [], []
        for r in range(world):
            c = Context(devices[r] if devices else 0)
            self.ctxs.append(c)
            c.set_fri_params(*fri_params)
            mine = []
            for t, bc, sp, bus in chips:
                a = c.air(bc, sp, t.shape[0], bus)
                f, n = shard_columns(t.shape[0], world, r)
                b = c.to_device(t[f:f + n]) if n else None
                self.airs.append(a)
                self.bufs.append(b)
                mine.append((a, b.ptr if b else 0, t.shape[1].bit_length() - 1, t.shape[0]))
            self.args.append(mine)

    def group(self):
        from powdr_b200 import Group
        g = Group(self.ctxs)
        self.groups.append(g)
        return g

    def launches(self):
        return [c.launch_count() for c in self.ctxs]

    def close(self):
        for g in self.groups:
            g.close()
        for a in self.airs:
            a.free()
        for b in self.bufs:
            if b is not None:
                b.free()
        for c in self.ctxs:
            c.close()


@pytest.fixture
def ranks():
    made = []

    def make(world, chips, **kw):
        made.append(Ranks(world, chips, **kw))
        return made[-1]

    yield make
    for r in made:
        r.close()


def _prove_rc(group, args, n_chips=None):
    """pb_prove_chips_group's return code for args (rank r's list of chips), bypassing the binding's own checks"""
    from powdr_b200.capi import Chip, ChipsProof
    K = len(args[0]) if n_chips is None else n_chips
    arrs = [(Chip * max(1, len(a)))(*[Chip(x.h.value if x else None, int(p or 0), int(ln), int(w)) for x, p, ln, w in a]) for a in args]
    ptrs = (C.c_void_p * len(arrs))(*[C.addressof(a) for a in arrs])
    cs = (C.c_uint32 * (4 * max(1, K)))()
    return group.lib.pb_prove_chips_group(group.h, ptrs, C.c_size_t(K), C.byref(ChipsProof()), cs)


def _stage_clocks_add_up(stats):
    for r, st in enumerate(stats):
        v = list(st["stage_ms"].values())
        assert len(v) == 12 and all(x >= 0 for x in v), (r, v)
        assert sum(v[:11]) == pytest.approx(v[11], rel=1e-5, abs=1e-3), (r, v)


@pytest.mark.parametrize("world", [2, 4, 8, 16])
@pytest.mark.parametrize("mix", range(len(MIXES)))
def test_group_equals_single_gpu_and_oracle(ctx, orc, world, mix):
    from powdr_b200 import VerifyingKey, verify_chips
    from powdr_b200.sharded import prove_chips_group
    spec = _raise(MIXES[mix], world)
    chips = _chips(spec, seed=mix)
    single = _single(ctx, chips)
    stats = [None] * world
    got = prove_chips_group(world, chips, stats=stats)
    assert len(got) == world and _same(got[0], single)
    _stage_clocks_add_up(stats)
    proof, cs, ys, q = single
    e_proof, e_cs, e_ys, e_q = orc.prove_chips(chips, n_queries=8, pow_bits=4)
    assert proof == e_proof and (cs == e_cs).all() and (ys == e_ys).all() and (q == e_q).all()
    assert orc.verify_chips(chips, proof, cs, ys, q, check_constraints=False) == 0
    # the library's verifier with the constraint identity: the chips with constraints get all-zero traces, which satisfy them
    zchips = _chips([s + (True,) if s[2] else s for s in spec], seed=mix)
    keys = [(VerifyingKey(bc, sp, t.shape[0], bus), t.shape[1].bit_length() - 1) for t, bc, sp, bus in zchips]
    zgot = prove_chips_group(world, zchips)[0]
    assert _same(zgot, _single(ctx, zchips))
    assert verify_chips(keys, *zgot, n_queries=8, pow_bits=4) == (0, 0)


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("small", ["2", "5", "7", "24"])
def test_fri_switch_point_does_not_change_the_group_proof(ctx, monkeypatch, world, small):
    """LDE heights 2^11, 2^9, 2^7, 2^6 (and 2^5 at world 2) on both sides of every switch point (test_gpu_sharded_chips.py)"""
    from powdr_b200.sharded import prove_chips_group
    spec = [(10, 9, 2, 3), (8, 7, 0, 4), (6, 6, 1, 2), (5, 5, 2, 0)] + ([(4, 4, 0, 3)] if world == 2 else [])
    chips = _chips(spec, seed=world)
    single = _single(ctx, chips)
    monkeypatch.setenv("PB_SHARD_FRI_SMALL", small)
    assert _same(prove_chips_group(world, chips)[0], single)


@pytest.mark.parametrize("world,lb", [(2, 1), (2, 2), (4, 1)])
def test_row_blocked_group_equals_the_resident_proof(ctx, world, lb):
    from powdr_b200.capi import footprint_bytes_sharded
    from powdr_b200.sharded import prove_chips_group
    chips = _chips(SPEC, seed=10 * world + lb)
    budget = footprint_bytes_sharded(_shapes(ctx, chips), world, lb)
    single = _single(ctx, chips)
    stats = [None] * world
    assert _same(prove_chips_group(world, chips, stats=stats, budget=budget)[0], single)
    assert [s["log_blocks"] for s in stats] == [lb] * world
    _stage_clocks_add_up(stats)


@pytest.mark.parametrize("n_queries", [1, 2, 3])
def test_row_blocked_query_phases_that_skip_sub_steps(ctx, n_queries):
    from powdr_b200.capi import footprint_bytes_sharded
    from powdr_b200.sharded import prove_chips_group
    world, lb = 2, 3
    chips = _chips(SPEC, seed=40 + n_queries)
    budget = footprint_bytes_sharded(_shapes(ctx, chips), world, lb)
    resident = prove_chips_group(world, chips, fri_params=(n_queries, 2))[0]
    stats = [None] * world
    blocked = prove_chips_group(world, chips, fri_params=(n_queries, 2), stats=stats, budget=budget)[0]
    assert [s["log_blocks"] for s in stats] == [lb] * world
    assert _same(blocked, resident)


def test_cross_rank_rules_are_refused_before_any_rank_starts(ranks):
    """different budgets, different FRI parameters, a chip's width or height that differs between ranks, ranks with different numbers of
    chips, the same context twice: PB_ERR_INVALID_ARG with no kernel launched on any context"""
    from powdr_b200 import Group
    from powdr_b200.capi import PbError
    chips = _chips([(6, 12, 2, 3), (5, 5, 1, 0)], seed=6)
    rk = ranks(2, chips)
    g = rk.group()
    before = rk.launches()
    a0, a1 = rk.args
    x = a1[1]
    refused = []
    rk.ctxs[1].set_memory_budget(1 << 30)
    refused.append(_prove_rc(g, rk.args))
    rk.ctxs[1].set_memory_budget(0)
    rk.ctxs[1].set_fri_params(8, 5)
    refused.append(_prove_rc(g, rk.args))
    rk.ctxs[1].set_fri_params(8, 4)
    refused.append(_prove_rc(g, [a0, [a1[0], (x[0], x[1], x[2], x[3] + 1)]]))
    refused.append(_prove_rc(g, [a0, [a1[0], (x[0], x[1], x[2] + 1, x[3])]]))
    for call in (lambda: g.prove_chips([a0, a1[:1]]), lambda: Group([rk.ctxs[0], rk.ctxs[0]])):
        with pytest.raises(PbError) as e:
            call()
        refused.append(e.value.code)
    assert refused == [INVALID] * 6
    assert rk.launches() == before


def test_a_rank_that_fails_alone_ends_the_call_on_every_rank(ctx, ranks):
    """rank 1 passes NULL for a chip whose columns it holds: its own check fails before its first collective while rank 0 goes on into
    the main commit's all-to-all.  The call returns rank 1's error with every stream idle (under a watchdog: a broken abort fails the
    test instead of hanging it), and the same group then proves the valid input"""
    import torch
    chips = _chips([(7, 12, 2, 3), (6, 6, 1, 0)], seed=7)
    rk = ranks(2, chips)
    g = rk.group()
    a0, a1 = rk.args
    x = a1[0]
    assert x[1]
    bad = [a0, [(x[0], 0, x[2], x[3]), a1[1]]]
    out = {}

    def call():
        out["rc"] = _prove_rc(g, bad)
        out["idle"] = torch.cuda.default_stream(0).query()        # the contexts run on device 0's default stream

    t = threading.Thread(target=call, daemon=True)
    t.start()
    t.join(timeout=300)
    assert not t.is_alive(), "pb_prove_chips_group did not return: a rank was left waiting"
    assert out == {"rc": INVALID, "idle": True}, out
    assert rk.ctxs[0].launch_count() > 0                            # rank 0 did start
    assert _same(g.prove_chips(rk.args), _single(ctx, chips))


def test_query_answers_only_for_the_groups_own_proof(ranks):
    chips = _chips([(6, 7, 2, 3), (5, 5, 1, 0)], seed=8)
    rk = ranks(2, chips)
    g = rk.group()
    lib = g.lib
    out = np.zeros(1 << 16, dtype=np.uint32)
    ptr, cap = out.ctypes.data_as(C.c_void_p), C.c_size_t(out.size)
    assert lib.pb_query_chips_group(g.h, ptr, cap, None, C.c_size_t(0)) == INVALID           # before any proof
    proof = g.prove_chips(rk.args)
    assert lib.pb_query_chips_group(g.h, ptr, cap, None, C.c_size_t(0)) == 0
    assert (out[:proof[3].size] == proof[3].ravel()).all()
    whole = [rk.ctxs[1].to_device(t) for t, _, _, _ in chips]                                  # rank 1's context proves on its own
    rk.ctxs[1].prove_chips([(a, w.ptr, ln, wd) for (a, _, ln, wd), w in zip(rk.args[1], whole)])
    assert lib.pb_query_chips_group(g.h, ptr, cap, None, C.c_size_t(0)) == INVALID
    assert _same(g.prove_chips(rk.args), proof)                                                 # a new group proof answers again
    assert lib.pb_query_chips_group(g.h, ptr, cap, None, C.c_size_t(0)) == 0


def _visible_gpus():
    import torch
    return torch.cuda.device_count()


@pytest.mark.parametrize("mix", [0, 1, 6])
def test_one_rank_per_gpu_equals_single_gpu(ctx, mix):
    n = _visible_gpus()
    if n < 2:
        pytest.skip("needs two or more GPUs")
    from powdr_b200.sharded import prove_chips_group
    world = 1 << (min(n, 16).bit_length() - 1)
    chips = _chips(_raise(MIXES[mix], world), seed=mix)
    assert _same(prove_chips_group(world, chips, devices=list(range(world)))[0], _single(ctx, chips))


KECCAK = (2022, 187, 1734)          # columns, constraints, interactions of the guest-keccak APC chip


def test_keccak_shape_at_2p20_rows_on_two_gpus_equals_the_single_gpu_proof():
    """2^20 x 2022 with 1734 interactions, one rank on each of two GPUs (resident at G = 2), equals the single-GPU proof"""
    import torch
    if _visible_gpus() < 2 or any(torch.cuda.get_device_properties(d).total_memory < (79 << 30) for d in range(2)):
        pytest.skip("needs two 80 GB-class GPUs")
    from powdr_b200 import Context
    from powdr_b200 import machine as M
    from powdr_b200.sharded import prove_chips_group
    from util import rand_field
    w, ncons, nints = KECCAK
    base = M.synthetic_machine(w, ncons, seed=21)
    mach = M.SymbolicMachine(base.constraints, M.synthetic_bus(base, nints, seed=22))
    bc, spans = M.compile_constraints(mach)
    bus = M.compile_bus(mach, 1)
    trace = rand_field(np.random.default_rng(20), (mach.width, 1 << 20))
    c = Context(0)
    try:
        c.set_fri_params(8, 4)
        air = c.air(bc, spans, mach.width, bus)
        d = c.to_device(trace)
        single = c.prove_chips([(air, d.ptr, 20, mach.width)])
        d.free()
        air.free()
    finally:
        c.close()
    torch.cuda.empty_cache()
    assert _same(prove_chips_group(2, [(trace, bc, spans, bus)], devices=[0, 1])[0], single)


def _demo_traces(log_n):
    """the traces examples/group_demo.c builds (its xorshift, canonical values)"""
    P, M64 = 2013265921, (1 << 64) - 1
    s = 88172645463325252
    out = []
    for c, ln in enumerate((log_n, log_n - 2)):
        n = 1 << ln
        t = np.zeros((3 if c == 0 else 5, n), dtype=np.uint32)
        for r in range(n):
            s ^= (s << 13) & M64
            s ^= s >> 7
            s ^= (s << 17) & M64
            if c == 0:
                a, b = s % 3, (s >> 8) % P
                t[:, r] = (a, b, a * b % P)
            else:
                x3, x4, x1 = s % P, (s >> 31) % P, (s >> 17) % P
                x0 = x3 * x4 % P
                t[:, r] = (x0, x1, (x0 + x1) % P, x3, x4)
        out.append(t)
    return out


def test_c_demo_proves_what_the_python_binding_proves(tmp_path):
    from powdr_b200 import Context
    lib_dir = os.path.join(ROOT, "powdr_b200", "_lib")
    exe = str(tmp_path / "group_demo")
    subprocess.check_call(["/usr/bin/gcc", "-std=c99", "-O2", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "examples", "group_demo.c"), "-L", lib_dir, "-lpowdr_b200", "-Wl,-rpath," + lib_dir, "-o", exe])
    log_n = 9
    r = subprocess.run([exe, str(log_n)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = {ln.split()[0]: ln.split()[1:] for ln in r.stdout.splitlines() if ln.strip()}
    assert lines["verify"] == ["0", "reason", "0"]
    OP_PUSH_APC, OP_PUSH_CONST, OP_ADD, OP_SUB, OP_MUL = 0, 1, 2, 3, 4
    bc0 = [OP_PUSH_APC, 0, OP_PUSH_APC, 1, OP_MUL, OP_PUSH_APC, 2, OP_SUB,
           OP_PUSH_APC, 0, OP_PUSH_APC, 0, OP_PUSH_CONST, 1, OP_SUB, OP_MUL, OP_PUSH_APC, 0, OP_PUSH_CONST, 2, OP_SUB, OP_MUL]
    bc1 = [OP_PUSH_APC, 0, OP_PUSH_APC, 1, OP_ADD, OP_PUSH_APC, 2, OP_SUB, OP_PUSH_APC, 3, OP_PUSH_APC, 4, OP_MUL, OP_PUSH_APC, 0, OP_SUB]
    traces = _demo_traces(log_n)
    c = Context(0)
    try:
        c.set_fri_params(4, 8)
        airs = [c.air(bc0, [(0, 8), (8, 14)], 3), c.air(bc1, [(0, 8), (8, 8)], 5)]
        bufs = [c.to_device(t) for t in traces]
        proof, _, _, q = c.prove_chips([(a, b.ptr, t.shape[1].bit_length() - 1, t.shape[0]) for a, b, t in zip(airs, bufs, traces)])
        for a in airs:
            a.free()
    finally:
        c.close()
    as_words = lambda v: [str(x) for x in v]                      # noqa: E731
    assert lines["main_root"] == as_words(proof["main_root"])
    assert lines["quotient_root"] == as_words(proof["quotient_root"])
    assert lines["zeta"] == as_words(proof["zeta"])
    assert lines["final_poly"] == as_words(np.ravel(proof["final_poly"]))
    assert lines["pow_witness"] == [str(proof["pow_witness"])]
    assert lines["query_rows"] == as_words(q[:, 0])
