"""LDE timing sweep over PB_LDE_BATCH x PB_LDE_STREAMS at the keccak shapes (run on the GPU box).

    python scripts/lde_sweep.py [width ...]        (default: 2022 main columns and the 3348-column permutation trace)
"""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import powdr_b200
log_n = 20
n = 1 << log_n
dev = torch.device("cuda", 0)
ctx = powdr_b200.Context(0, torch.cuda.current_stream().cuda_stream)
CONFIGS = [(None, None), (66, 1), (33, 1), (16, 1), (8, 1), (4, 1), (16, 2), (8, 2), (4, 2), (8, 4), (4, 4), (3, 4), (2, 4),
           (4, 8), (2, 8)]
for w in [int(a) for a in sys.argv[1:]] or [2022, 3348]:
    trace = torch.randint(0, powdr_b200.P, (w, n), dtype=torch.int32, device=dev)
    out = torch.empty((w, 2 * n), dtype=torch.int32, device=dev)
    ref = None
    for batch, streams in CONFIGS * 2:          # two passes over the list: the repeat shows the run-to-run spread
        for k, v in (("PB_LDE_BATCH", batch), ("PB_LDE_STREAMS", streams)):
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = str(v)
        for _ in range(2):
            ctx.lde_batch(trace.data_ptr(), log_n, w, out.data_ptr())
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(3):
            ctx.lde_batch(trace.data_ptr(), log_n, w, out.data_ptr())
        e1.record()
        torch.cuda.synchronize()
        chk = int(out[::97, ::4099].to(torch.int64).sum().item())
        ref = chk if ref is None else ref
        print("width %d batch %7s streams %7s: %.2f ms  %s" % (w, batch or "default", streams or "default", e0.elapsed_time(e1) / 3,
                                                             "ok" if chk == ref else "MISMATCH"), flush=True)
    del trace, out
    torch.cuda.empty_cache()
