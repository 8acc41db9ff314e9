"""Per-kernel timing of the coset LDE (Context.lde_batch, blowup 2) at the keccak shapes, under torch.profiler (run on the GPU box).

Nsight does not run where this project is measured, so this is how each pass's share of the LDE is taken.  For every kernel it
prints the device time per LDE call, the algorithmic HBM traffic of that pass over its time (against the data-sheet 3.35 TB/s of
an H100 SXM), and radix-2 butterflies per SM clock per SM.  The card name, power limit and SM clocks are printed in the same run.

    python scripts/lde_kernels.py [--log-n 20] [--widths 2022,3348] [--calls 3]
"""
import argparse
import os
import re
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch.profiler import ProfilerActivity, profile

import powdr_b200

HBM_BPS = 3.35e12        # H100 SXM data sheet


def smi(fields):
    out = subprocess.run(["nvidia-smi", "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0],
                          "--query-gpu=" + fields, "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip() or out.stderr.strip()


def pass_work(name, n, blowup):
    """(label, words moved per column element, radix-2 butterflies per column) of one LDE pass, from the kernel's name"""
    n_lo = n if n <= 10 else (n + 1) // 2
    n_hi = n - n_lo
    N, B = 1 << n, 1 << blowup
    inv = "true" in name.split("(")[0] or "transposed_tma_kernel" in name      # the TMA kernel of that name is K2a only
    if "strided" in name:
        return ("K1 inverse high bits", 2, N // 2 * n_hi) if inv else ("K3 forward high bits", 2 * B, B * (N // 2) * n_hi)
    if "lde_low_bits" in name:
        return ("K2a+K2b low bits, fused", 1 + B, (1 + B) * (N // 2) * n_lo)
    if "transposed" in name:
        return ("K2a inverse low bits", 2, N // 2 * n_lo) if inv else ("K2b forward low bits", 1 + B, B * (N // 2) * n_lo)
    return ("other", 0, 0)


def device_us(evt):
    for attr in ("device_time_total", "cuda_time_total"):
        if hasattr(evt, attr):
            return getattr(evt, attr)
    raise RuntimeError("profiler event has no device time")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=20)
    ap.add_argument("--widths", default="2022,3348")
    ap.add_argument("--calls", type=int, default=3)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    props = torch.cuda.get_device_properties(dev)
    n_sms = props.multi_processor_count
    print("card:", smi("name,power.limit,clocks.sm,clocks.max.sm"), "| SMs", n_sms, flush=True)
    sm_hz = float(re.findall(r"\d+", smi("clocks.max.sm"))[0]) * 1e6      # butterflies/clk/SM below are at the maximum SM clock
    ctx = powdr_b200.Context(0, torch.cuda.current_stream().cuda_stream)
    n, blowup = args.log_n, 1
    for w in [int(x) for x in args.widths.split(",")]:
        trace = torch.randint(0, powdr_b200.P, (w, 1 << n), dtype=torch.int32, device=dev)
        out = torch.empty((w, (1 << n) << blowup), dtype=torch.int32, device=dev)
        for _ in range(2):
            ctx.lde_batch(trace.data_ptr(), n, w, out.data_ptr(), log_blowup=blowup)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.calls):
            ctx.lde_batch(trace.data_ptr(), n, w, out.data_ptr(), log_blowup=blowup)
        e1.record()
        torch.cuda.synchronize()
        wall = e0.elapsed_time(e1) / args.calls
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.calls):
                ctx.lde_batch(trace.data_ptr(), n, w, out.data_ptr(), log_blowup=blowup)
            torch.cuda.synchronize()
        print("2^%d x %d: %.2f ms per LDE (events, profiler off), sm clock now: %s" % (n, w, wall, smi("clocks.sm")), flush=True)
        tot = 0.0
        for evt in sorted(prof.key_averages(), key=lambda e: -device_us(e)):
            if device_us(evt) <= 0:
                continue
            ms = device_us(evt) / 1e3 / args.calls
            tot += ms
            label, words, bfly = pass_work(evt.key, n, blowup)
            gbs = words * 4 * (w << n) / (ms / 1e3) if words else 0.0
            rate = bfly * w / (ms / 1e3) / sm_hz / n_sms if bfly else 0.0
            print("  %8.2f ms  %5.0f GB/s (%4.1f %% of HBM)  %6.2f butterflies/clk/SM  launches %4d  %-22s %s"
                  % (ms, gbs / 1e9, 100 * gbs / HBM_BPS, rate, evt.count // args.calls, label, evt.key[:90]), flush=True)
        print("  %8.2f ms  summed kernel time per LDE" % tot, flush=True)
        del trace, out
        torch.cuda.empty_cache()
    ctx.close()


if __name__ == "__main__":
    main()
