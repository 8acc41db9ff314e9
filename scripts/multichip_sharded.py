#!/usr/bin/env python3
"""The 50-chip segment of `bench.py --workload multichip --one-transcript` proved under ONE transcript across N GPUs
(pb_prove_chips_sharded + pb_query_chips_sharded), one JSON line per run.

  torchrun --nproc-per-node N scripts/multichip_sharded.py   # N ranks over NCCL (TorchComm); N = 1 times pb_prove_chips instead
  python scripts/multichip_sharded.py --threads G             # G thread-ranks on one GPU (ThreadComm): counts only, no speed

Chips are bench.multichip_shapes() with bench.py's seeds, so the traces are the ones `--workload multichip --one-transcript`
proves; --chips K takes the first K shapes.  Rank 0 also proves the gathered traces once with pb_prove_chips and reports whether
the proof, the cumulative sums, the opened values and the queries are equal word for word (proof_equals_single_gpu)."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

P = 2013265921


def card():
    import torch
    name = torch.cuda.get_device_name()
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        power = float(out.splitlines()[0])
    except Exception:       # noqa: BLE001 -- the number is reported beside the timing, not needed for it
        power = None
    return name, power


def make_chips(ctx, a, dev):
    """[(air, full device trace (torch), log_n, width, bytecode, spans, bus)] of the first a.chips shapes, seeded as bench.py"""
    import torch
    import bench
    from powdr_b200 import machine as M
    out = []
    for i, (ln, w, c) in enumerate(bench.multichip_shapes()[:a.chips]):
        base = M.synthetic_machine(w, c, seed=0xEC000 + i)
        n_ints = 0 if a.no_interactions else max(1, (w * 1734) // 2022)
        mach = M.SymbolicMachine(base.constraints, M.synthetic_bus(base, n_ints, seed=0xEC200 + i)) if n_ints else base
        bc, spans = M.compile_constraints(mach)
        bus = M.compile_bus(mach, 1) if n_ints else None
        gen = torch.Generator(device=dev)
        gen.manual_seed(0xEC100 + i)
        tr = torch.randint(0, P, (mach.width, 1 << ln), dtype=torch.int32, device=dev, generator=gen)
        out.append((ctx.air(bc, spans, mach.width, bus) if ctx else None, tr, ln, mach.width, bc, spans, bus))
    return out


def run_threads(a):
    """G thread-ranks on one GPU: collectives, bytes, launches and host synchronisations of one proof + query phase"""
    import numpy as np
    import torch
    from powdr_b200.sharded import prove_chips_threads
    chips = make_chips(None, a, torch.device("cuda", 0))
    host = [(tr.cpu().numpy().view(np.uint32), bc, spans, bus) for _, tr, _, _, bc, spans, bus in chips]
    del chips
    torch.cuda.empty_cache()
    stats = [None] * a.threads
    res = prove_chips_threads(a.threads, host, fri_params=(a.queries, a.pow_bits), stats=stats)
    name, power = card()
    print(json.dumps({"mode": "threads", "world": a.threads, "chips": len(host), "interactions": not a.no_interactions,
                      "collective_calls": stats[0]["calls"], "collective_bytes_per_rank": stats[0]["bytes"],
                      "gpu_launches": [s["launches"] for s in stats], "ranks_agree": all(r[0] == res[0][0] for r in res),
                      "card": name, "power_limit_w": power}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--chips", type=int, default=50)
    ap.add_argument("--no-interactions", action="store_true")
    ap.add_argument("--threads", type=int, default=0, help="G thread-ranks on one GPU (counts only)")
    ap.add_argument("--queries", type=int, default=100)
    ap.add_argument("--pow-bits", type=int, default=16)
    a = ap.parse_args()
    if a.threads:
        return run_threads(a)
    import torch
    import powdr_b200
    from powdr_b200.sharded import TorchComm, shard_columns
    world, rank = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist = None
    if world > 1:
        import torch.distributed as dist
        os.environ.setdefault("NCCL_DEBUG_FILE", "/dev/stderr")
        dist.init_process_group("nccl", device_id=dev)
    stream = torch.cuda.current_stream()
    ctx = powdr_b200.Context(local, stream.cuda_stream)
    ctx.set_fri_params(a.queries, a.pow_bits)
    chips = make_chips(ctx, a, dev)
    comm = TorchComm() if world > 1 else None
    blocks, args = [], []
    for air, tr, ln, w, *_ in chips:
        if comm:
            first, count = shard_columns(w, world, rank)
            blk = tr[first:first + count].contiguous()
            blocks.append(blk)
            args.append((air, blk.data_ptr() if count else 0, ln, w))
        else:
            args.append((air, tr.data_ptr(), ln, w))

    def step():
        return ctx.prove_chips_sharded(args, comm) if comm else ctx.prove_chips(args)

    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    calls0, l0 = (comm.calls, comm.bytes) if comm else (0, 0), ctx.launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(a.steps):
        res = step()
    e1.record(stream)
    torch.cuda.synchronize()
    t = torch.tensor([e0.elapsed_time(e1)], dtype=torch.float64, device=dev)
    if dist:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    out = {"mode": "torchrun" if comm else "single", "world": world, "chips": len(chips), "interactions": not a.no_interactions,
           "ms_per_step": float(t.item()) / a.steps, "stages_ms": ctx.last_stage_ms(),
           "gpu_launches_per_step": (ctx.launch_count() - l0) / a.steps}
    if comm:
        out["collective_calls_per_step"] = (comm.calls - calls0[0]) / a.steps
        out["collective_bytes_per_rank_per_step"] = (comm.bytes - calls0[1]) / a.steps
    if rank == 0:
        if comm:
            single = ctx.prove_chips([(air, tr.data_ptr(), ln, w) for air, tr, ln, w, *_ in chips])
            out["proof_equals_single_gpu"] = bool(res[0] == single[0] and (res[1] == single[1]).all() and (res[2] == single[2]).all()
                                                  and (res[3] == single[3]).all())
        out["card"], out["power_limit_w"] = card()
        print(json.dumps(out), flush=True)
    if dist:
        dist.barrier()
        dist.destroy_process_group()
    ctx.close()


if __name__ == "__main__":
    main()
