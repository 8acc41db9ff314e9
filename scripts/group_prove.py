#!/usr/bin/env python3
"""pb_prove_chips_group (+ pb_query_chips_group) timed against pb_prove_chips on one GPU, one JSON line per world.

  python scripts/group_prove.py [--steps 5] [--log-n 20] [--worlds 2 4 8]

With two or more visible GPUs: the keccak LogUp shape (2022 columns, 187 constraints, 1734 interactions, 100 queries, 16 proof-of-work
bits) at 2^--log-n rows, one rank per GPU at G = 2, 4, 8 up to the number visible; the single-GPU proof is timed first and freed.
With one GPU: a HARNESS COMPARISON, not a multi-GPU number: G thread-ranks on that GPU through the group (device-to-device copies) and
through ThreadComm (host staging around every collective), alternated with pb_prove_chips, at a small shape (--small-log-n, --small-width).
Every time is the median wall time of --steps runs after one warm-up of each; each run includes the query phase.  The card name and
power limit go beside the times, and the exchange bytes per rank are computed from the shapes."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WIDTH, CONSTRAINTS, INTERACTIONS = 2022, 187, 1734


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True,
                             timeout=20).stdout.strip()
        power = float(out.splitlines()[0])
    except Exception:       # noqa: BLE001 -- reported beside the timing, not needed for it
        power = None
    return name, power


def exchange_bytes(log_n, width, perm_width, world):
    """bytes each rank receives in one resident proof's four large all-to-alls: the main LDE, the LogUp rows, the permutation columns
    back and the permutation LDE ((G - 1) / G of it crosses between ranks)"""
    n = 1 << log_n
    per, perp = -(-width // world), -(-perm_width // world)
    return {"main_lde": 8 * n * per, "logup_rows": 4 * n * per if perm_width else 0, "perm_back": 4 * n * perp, "perm_lde": 8 * n * perp}


def segment(log_n, width, constraints, interactions, seed):
    import numpy as np
    from powdr_b200 import machine as M
    base = M.synthetic_machine(width, constraints, seed=seed)
    mach = M.SymbolicMachine(base.constraints, M.synthetic_bus(base, interactions, seed=seed + 1))
    bc, spans = M.compile_constraints(mach)
    bus = M.compile_bus(mach, 1)
    trace = np.random.default_rng(seed).integers(0, 2013265921, size=(mach.width, 1 << log_n), dtype=np.uint32)
    return trace, bc, spans, bus


class Ranks:
    """world contexts (rank r on devices[r]) with the AIR and rank r's column block of the trace"""

    def __init__(self, world, chip, devices, fri):
        from powdr_b200 import Context
        from powdr_b200.sharded import shard_columns
        trace, bc, spans, bus = chip
        self.ctxs, self.airs, self.bufs, self.args = [], [], [], []
        for r in range(world):
            c = Context(devices[r])
            c.set_fri_params(*fri)
            a = c.air(bc, spans, trace.shape[0], bus)
            f, n = shard_columns(trace.shape[0], world, r)
            b = c.to_device(trace[f:f + n]) if n else None
            self.ctxs.append(c)
            self.airs.append(a)
            self.bufs.append(b)
            self.args.append([(a, b.ptr if b else 0, trace.shape[1].bit_length() - 1, trace.shape[0])])

    def close(self):
        for a in self.airs:
            a.free()
        for b in self.bufs:
            if b is not None:
                b.free()
        for c in self.ctxs:
            c.close()


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return (time.perf_counter() - t0) * 1e3, out


def single_runner(chip, fri):
    from powdr_b200 import Context
    trace, bc, spans, bus = chip
    c = Context(0)
    c.set_fri_params(*fri)
    a = c.air(bc, spans, trace.shape[0], bus)
    d = c.to_device(trace)
    run = lambda: c.prove_chips([(a, d.ptr, trace.shape[1].bit_length() - 1, trace.shape[0])])     # noqa: E731

    def close():
        d.free()
        a.free()
        c.close()
    return run, close, a.perm_width


def thread_comm_runner(rk):
    """one pb_prove_chips_sharded + pb_query_chips_sharded per rank on its own thread, collectives through ThreadComm"""
    from powdr_b200.sharded import ThreadComm, ThreadGroup
    world = len(rk.ctxs)

    def run():
        tg = ThreadGroup(world)
        out = [None] * world
        comms = [ThreadComm(tg, r, rk.ctxs[r]) for r in range(world)]

        def body(r):
            out[r] = rk.ctxs[r].prove_chips_sharded(rk.args[r], comms[r])
        ts = [threading.Thread(target=body, args=(r,)) for r in range(world)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        return out[0]
    return run


def same(a, b):
    return a[0] == b[0] and (a[1] == b[1]).all() and (a[2] == b[2]).all() and (a[3] == b[3]).all()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--log-n", type=int, default=20)
    ap.add_argument("--worlds", type=int, nargs="+", default=[2, 4, 8])
    ap.add_argument("--small-log-n", type=int, default=16)
    ap.add_argument("--small-width", type=int, default=256)
    a = ap.parse_args()
    import torch
    from powdr_b200 import Group
    n_gpus = torch.cuda.device_count()
    name, power = card()
    multi = n_gpus >= 2
    if multi:
        log_n, fri = a.log_n, (100, 16)
        chip = segment(log_n, WIDTH, CONSTRAINTS, INTERACTIONS, seed=20)
        worlds = [w for w in a.worlds if w <= n_gpus]
    else:
        log_n, fri = a.small_log_n, (100, 16)
        chip = segment(log_n, a.small_width, a.small_width // 8, a.small_width // 2, seed=20)
        worlds = [w for w in a.worlds if w <= 4]
    run_single, close_single, perm_width = single_runner(chip, fri)
    if multi:                                   # the single-GPU proof first, then freed: device 0 also holds rank 0
        run_single()
        t_single = [timed(run_single)[0] for _ in range(a.steps)]
        want = run_single()
        close_single()
        torch.cuda.empty_cache()
    for world in worlds:
        rk = Ranks(world, chip, list(range(world)) if multi else [0] * world, fri)
        g = Group(rk.ctxs)
        try:
            run_group = lambda: g.prove_chips(rk.args)      # noqa: E731
            runs = {"group": run_group}
            if not multi:
                runs["single"] = run_single
                runs["thread_comm"] = thread_comm_runner(rk)
            outs = {k: f() for k, f in runs.items()}        # warm-up of each
            times = {k: [] for k in runs}
            for _ in range(a.steps):                        # alternated
                for k, f in runs.items():
                    times[k].append(timed(f)[0])
            ref = want if multi else outs["single"]
            line = {"card": name, "power_limit_w": power, "gpus_visible": n_gpus, "world": world, "ranks_on": "one GPU each" if multi else "GPU 0",
                    "kind": "multi-GPU" if multi else "harness comparison on one GPU, not a multi-GPU number",
                    "shape": {"log_n": log_n, "width": chip[0].shape[0], "interactions": INTERACTIONS if multi else a.small_width // 2,
                              "perm_width": perm_width, "queries": fri[0], "pow_bits": fri[1]},
                    "exchange_bytes_per_rank": exchange_bytes(log_n, chip[0].shape[0], perm_width, world),
                    "median_ms": {k: round(statistics.median(v), 2) for k, v in times.items()},
                    "group_equals_single_gpu": bool(same(outs["group"], ref))}
            if multi:
                line["median_ms"]["single"] = round(statistics.median(t_single), 2)
            else:
                line["thread_comm_equals_single_gpu"] = bool(same(outs["thread_comm"], ref))
            print(json.dumps(line), flush=True)
        finally:
            g.close()
            rk.close()
    if not multi:
        close_single()


if __name__ == "__main__":
    main()
