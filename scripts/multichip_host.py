#!/usr/bin/env python3
"""The 50-chip segment of `bench.py --workload multichip --one-transcript` proved under one transcript on one GPU, from three places,
runs alternated, one JSON line with the medians:

  device   pb_prove_chips on device-resident traces (what the benchmark times)
  host     pb_prove_chips_host from pinned host memory: the copies stream behind the LDE and the leaf hashing
  serial   the H2D copy of every chip from the same pinned memory, then pb_prove_chips

Each time is a host clock around one call that ends in a device synchronise (the proof and the opened values; no query phase).  Chips
are bench.multichip_shapes() with bench.py's seeds; --chips K takes the first K.  The first round also checks that the three proofs are
equal word for word (proofs_equal).  The card's name, power limit and SM clock are read in the same run.

  python scripts/multichip_host.py [--runs 3] [--chips 50]"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def card():
    import torch
    q = "power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader,nounits", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=20).stdout.strip().splitlines()[0]
        power, sm, sm_max = [float(x) for x in out.split(",")]
    except Exception:       # noqa: BLE001 -- reported beside the timing, not needed for it
        power = sm = sm_max = None
    return {"card": torch.cuda.get_device_name(), "power_limit_w": power, "sm_clock_mhz": sm, "sm_clock_max_mhz": sm_max}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--chips", type=int, default=50)
    ap.add_argument("--queries", type=int, default=100)
    ap.add_argument("--pow-bits", type=int, default=16)
    a = ap.parse_args()
    log = lambda *m: print(*m, file=sys.stderr, flush=True)         # progress: the AIRs of 50 chips take a while to compile
    import torch
    import powdr_b200
    from multichip_sharded import make_chips
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    ctx = powdr_b200.Context(0, torch.cuda.current_stream().cuda_stream)
    ctx.set_fri_params(a.queries, a.pow_bits)
    a.no_interactions = False
    chips = make_chips(ctx, a, dev)
    log("compiled and generated %d chips" % len(chips))
    host = []                                             # pinned copies of the device traces
    for _, tr, _, _, _, _, _ in chips:
        nbytes = tr.numel() * 4
        p = ctx.host_alloc(nbytes)
        words = tr.cpu().numpy()                          # held until the copy below is done
        C.memmove(p, words.ctypes.data, nbytes)
        host.append((p, nbytes))
    torch.cuda.synchronize()
    dev_args = [(air, tr.data_ptr(), ln, w) for air, tr, ln, w, _, _, _ in chips]
    host_args = [(air, p, ln, w) for (air, _, ln, w, _, _, _), (p, _) in zip(chips, host)]

    def device():
        return ctx.prove_chips(dev_args, want_queries=False)

    def from_host():
        return ctx.prove_chips(host_args, want_queries=False, on_device=False)

    def serial():
        for (_, tr, _, _, _, _, _), (p, nbytes) in zip(chips, host):
            assert ctx.lib.pb_copy_h2d(ctx.h, C.c_void_p(tr.data_ptr()), C.c_void_p(p), C.c_size_t(nbytes)) == 0
        return ctx.prove_chips(dev_args, want_queries=False)

    modes = {"device": device, "host": from_host, "serial": serial}
    times = {k: [] for k in modes}
    blocks = {}
    out = {}
    for k, f in modes.items():                            # warm-up: twiddles, JIT modules, workspaces
        out[k] = f()
        blocks[k] = ctx.last_row_blocks()
        log("warm-up", k)
    same = all(out[k][0] == out["device"][0] and all((x == y).all() for x, y in zip(out[k][1:3], out["device"][1:3])) for k in modes)
    stages = {}
    for _ in range(a.runs):
        for k, f in modes.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            f()
            torch.cuda.synchronize()
            times[k].append(1e3 * (time.perf_counter() - t0))
            stages[k] = ctx.last_stage_ms()
            log(k, round(times[k][-1], 1), "ms")
    for p, _ in host:
        ctx.host_free(p)
    res = {"chips": len(chips), "trace_gb": sum(n for _, n in host) / 1e9, "runs": a.runs, "queries": a.queries, "pow_bits": a.pow_bits,
           "median_ms": {k: statistics.median(v) for k, v in times.items()}, "runs_ms": times, "row_blocks": blocks, "proofs_equal": same,
           "stage_ms_last": {k: {s: round(v, 2) for s, v in st.items()} for k, st in stages.items()}}
    res.update(card())
    print(json.dumps(res))


if __name__ == "__main__":
    main()
