#!/usr/bin/env python3
"""The keccak APC shape (2022 columns, 187 constraints, 1734 interactions) proved on N GPUs by pb_prove_chips_sharded, resident and with
each rank block in row sub-blocks (a memory budget on every rank), one JSON line per shape from rank 0.

  torchrun --nproc-per-node 2 scripts/sharded_row_blocks.py [--log-n 20 21] [--steps 5] [--blocks 2]

Per shape: the resident and the blocked proof alternate for --steps rounds after a warm-up of each, and the medians are reported
(resident only where its footprint fits the card).  The blocked path is forced by the budget pb_footprint_bytes_sharded gives for
--blocks sub-blocks, or for the fewest above that which fit the card beside the column share.  all_to_all_bytes_per_rank are computed
from the shapes (the send buffers of every all-to-all of one proof, the query phase left out); collective_bytes_per_rank are what
TorchComm counted, query phase included.  The card name and power limit go beside
the times."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

P = 2013265921
WIDTH, CONSTRAINTS, INTERACTIONS = 2022, 187, 1734


def card():
    import torch
    name = torch.cuda.get_device_name()
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        power = float(out.splitlines()[0])
    except Exception:       # noqa: BLE001 -- reported beside the timing, not needed for it
        power = None
    return name, power


def all_to_all_bytes(log_n, width, perm_width, world, lb):
    """bytes one rank sends through all-to-alls in one proof (before its query phase): resident, the main LDE, the LogUp rows there and
    back, the permutation LDE; blocked (lb > 0), the main and permutation sub-steps of the two commits, the quotient and the reduced
    opening instead of the two LDE exchanges"""
    n = 1 << log_n
    ms, per, perp = 2 * n // world, -(-width // world), -(-perm_width // world)
    rows = per * n + perp * n                                           # LogUp: my columns' rows out, my rows' perm columns back
    if not lb:
        return 4 * (world * per * ms + rows + world * perp * ms)
    return 4 * (3 * world * per * ms + rows + 3 * world * perp * ms)   # B sub-steps of ms / B rows, three phases each


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, nargs="+", default=[20, 21])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--blocks", type=int, default=2, help="log2 of the sub-blocks of the blocked runs")
    ap.add_argument("--queries", type=int, default=100)
    ap.add_argument("--pow-bits", type=int, default=16)
    a = ap.parse_args()
    import torch
    import torch.distributed as dist
    import powdr_b200
    from powdr_b200 import machine as M
    from powdr_b200.capi import footprint_bytes_sharded
    from powdr_b200.sharded import TorchComm, shard_columns
    world, rank = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0"))
    if world < 2:
        sys.exit("run under torchrun with --nproc-per-node 2 or more")
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    stream = torch.cuda.current_stream()
    ctx = powdr_b200.Context(local, stream.cuda_stream)
    ctx.set_fri_params(a.queries, a.pow_bits)
    base = M.synthetic_machine(WIDTH, CONSTRAINTS, seed=0x5B)
    mach = M.SymbolicMachine(base.constraints, M.synthetic_bus(base, INTERACTIONS, seed=0x5C))
    bc, spans = M.compile_constraints(mach)
    air = ctx.air(bc, spans, mach.width, M.compile_bus(mach, 1))
    comm = TorchComm()
    total = torch.cuda.get_device_properties(dev).total_memory
    for log_n in a.log_n:
        first, count = shard_columns(mach.width, world, rank)
        gen = torch.Generator(device=dev)
        gen.manual_seed(0x5D00 + log_n)
        block = torch.randint(0, P, (mach.width, 1 << log_n), dtype=torch.int32, device=dev, generator=gen)[first:first + count].contiguous()
        torch.cuda.empty_cache()
        args = [(air, block.data_ptr(), log_n, mach.width)]
        shape = [(log_n, mach.width, air.perm_width)]
        share = block.numel() * 4
        room = total - share - (1 << 30)                                # 1 GiB for the CUDA context and NCCL
        resident_fits = footprint_bytes_sharded(shape, world, 0) <= room
        lb = a.blocks
        while footprint_bytes_sharded(shape, world, lb) > room and world << (lb + 1) <= 16:
            lb += 1
        budget = footprint_bytes_sharded(shape, world, lb)
        runs = {"blocked": budget}
        if resident_fits:
            runs["resident"] = 0
        times, calls = {k: [] for k in runs}, {}
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for step in range(a.steps + 1):                                 # step 0 warms each path up
            for kind, b in runs.items():
                ctx.set_memory_budget(b)
                b0 = comm.bytes
                e0.record(stream)
                res = ctx.prove_chips_sharded(args, comm)
                e1.record(stream)
                torch.cuda.synchronize()
                t = torch.tensor([e0.elapsed_time(e1)], dtype=torch.float64, device=dev)
                dist.all_reduce(t, op=dist.ReduceOp.MAX)
                if step:
                    times[kind].append(float(t.item()))
                calls[kind] = (comm.bytes - b0, ctx.last_row_blocks())
        del res, block
        if rank == 0:
            name, power = card()
            out = {"shape": "2^%d x %d, %d interactions" % (log_n, mach.width, INTERACTIONS), "world": world, "perm_width": air.perm_width,
                   "ms_median": {k: statistics.median(v) for k, v in times.items()}, "ms_all": times,
                   "log_blocks": {k: v[1] for k, v in calls.items()}, "collective_bytes_per_rank": {k: v[0] for k, v in calls.items()},
                   "all_to_all_bytes_per_rank": {k: all_to_all_bytes(log_n, mach.width, air.perm_width, world, lb if k == "blocked" else 0)
                                                 for k in runs},
                   "footprint_bytes_per_rank": {k: footprint_bytes_sharded(shape, world, lb if k == "blocked" else 0) for k in runs},
                   "card": name, "power_limit_w": power}
            print(json.dumps(out), flush=True)
        torch.cuda.empty_cache()
    air.free()
    dist.barrier()
    dist.destroy_process_group()
    ctx.close()


if __name__ == "__main__":
    main()
