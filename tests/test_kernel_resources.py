"""CPU test of what the compiler made of the hot kernels: every LDE pass (nttf::, ntttma::) and the leaf hash keep their working
set in registers.  A stack frame there means an unrolled register array (x[32] of a 5-stage butterfly round) went to local
memory, which made the sm_90a LDE passes several times slower with identical results -- only the resource table shows it."""
import os
import re
import subprocess

from powdr_b200 import build

CHECKED = {"_ZN4nttf": "nttf::", "_ZN6ntttma": "ntttma::", "_ZN2p221leaf_hash_cols_kernel": "p2::leaf_hash_cols_kernel"}


def resource_usage():
    lib = build.build()
    cuobjdump = os.path.join(os.path.dirname(build.NVCC), "cuobjdump")
    out = subprocess.run([cuobjdump, "-res-usage", lib], check=True, capture_output=True, text=True).stdout
    rows = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    return {name: (int(reg), int(stack), int(local)) for name, reg, stack, local in rows}


def test_every_lde_pass_and_leaf_kernel_has_no_stack_frame_or_local_memory():
    usage = resource_usage()
    checked = {name: u for name, u in usage.items() if name.startswith(tuple(CHECKED))}
    per_prefix = {p: sum(name.startswith(p) for name in checked) for p in CHECKED}
    # strided (n_hi, n_lo) for log_n 11..24: 14 x 2 directions; transposed n_lo = 1..12: 12 x 2 directions; 2 TMA passes; the leaf hash
    assert per_prefix == {"_ZN4nttf": 52, "_ZN6ntttma": 2, "_ZN2p221leaf_hash_cols_kernel": 1}, per_prefix
    bad = {name: "REG %d STACK %d LOCAL %d" % u for name, u in checked.items() if u[1] or u[2]}
    assert not bad, bad
