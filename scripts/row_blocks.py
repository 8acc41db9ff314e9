"""Time the single-GPU segment proof of the keccak LogUp shape (2^20 rows, the 1734-interaction AIR over 1963 of 2022 columns, 3348
permutation columns) resident against 2, 4 and 8 row blocks (pb_ctx_set_memory_budget from pb_footprint_bytes), alternated, median of
--reps, and the 2^21-row shape in 8 row blocks; checks that every blocked proof equals the resident one.  Prints one JSON object with
the card name and power limit read in the same run (and writes it to --out, if given)."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

P = 2013265921


def card():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [x.strip() for x in out.splitlines()[0].split(",")])) if out else {}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--lbs", default="1,2,3")
    ap.add_argument("--big", type=int, default=1, help="proofs of the 2^21 shape (0: skip)")
    ap.add_argument("--out", default=None, help="also write the JSON object to this file")
    a = ap.parse_args()
    import ctypes as C

    import torch

    from powdr_b200 import build, capi
    from powdr_b200 import machine as M
    build.build()
    ctx = capi.Context(0)
    mach = M.SymbolicMachine([], M.synthetic_bus(2022, 1734, seed=0xB2000002))
    w = mach.width
    air = ctx.air([], [], w, M.compile_bus(mach, 1))
    res = {"card": card(), "width": w, "perm_width": air.perm_width, "n_queries": ctx.n_queries}

    def trace_of(log_n):
        t = torch.randint(0, P, (w, 1 << log_n), dtype=torch.int32, device="cuda",
                          generator=torch.Generator(device="cuda").manual_seed(log_n))
        assert ctx.lib.pb_to_monty(ctx.h, C.c_void_p(t.data_ptr()), C.c_size_t(t.numel())) == 0
        torch.cuda.synchronize()
        return t

    def prove(t, log_n, lb):
        ctx.set_memory_budget(capi.footprint_bytes([(log_n, w, air.perm_width)], lb) if lb else 0)
        t0 = time.perf_counter()
        proof = ctx.prove_segment(air, t.data_ptr(), log_n, w, on_device=True)
        ms = 1e3 * (time.perf_counter() - t0)
        assert ctx.last_row_blocks() == lb, (ctx.last_row_blocks(), lb)
        return proof, ms, ctx.last_stage_ms()

    lbs = [0] + [int(x) for x in a.lbs.split(",")]
    t = trace_of(20)
    ref = prove(t, 20, 0)[0]                              # warm-up: JIT, twiddles, workspaces
    for lb in lbs[1:]:
        assert prove(t, 20, lb)[0] == ref, lb
    times = {lb: [] for lb in lbs}
    stages = {}
    for _ in range(a.reps):
        for lb in lbs:
            proof, ms, st = prove(t, 20, lb)
            assert proof == ref, lb
            times[lb].append(ms)
            stages[lb] = st
    res["log_n_20"] = {str(1 << lb): {"median_ms": statistics.median(v), "ms": v, "stages_ms": stages[lb]} for lb, v in times.items()}
    del t
    torch.cuda.empty_cache()
    if a.big:
        t = trace_of(21)
        runs = [prove(t, 21, 3) for _ in range(a.big + 1)]      # the first one warms up
        assert all(r[0] == runs[0][0] for r in runs)
        res["log_n_21"] = {"8": {"ms": [r[1] for r in runs[1:]], "stages_ms": runs[-1][2]}}
        del t
    ctx.set_memory_budget(0)
    air.free()
    ctx.close()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
