"""CPU checks of the K-chip sharded prover: its NULL-argument checks need no device, and its chip-table transposes keep their working
set in registers (cuobjdump -res-usage, as test_kernel_resources.py does for the LDE passes)."""
import ctypes as C

from test_kernel_resources import resource_usage


def test_null_arguments_are_refused_without_a_device():
    from powdr_b200.capi import Chip, ChipsProof, load_library
    lib = load_library()
    proof, cs = ChipsProof(), (C.c_uint32 * 4)()
    arr = (Chip * 1)(Chip(None, None, 8, 4))
    assert lib.pb_prove_chips_sharded(None, arr, C.c_size_t(1), None, C.byref(proof), cs) == -1
    assert lib.pb_query_chips_sharded(None, None, None, C.c_size_t(0), None, C.c_size_t(0)) == -1


def test_chip_table_kernels_have_no_stack_frame_or_local_memory():
    usage = resource_usage()
    names = {n: u for n, u in usage.items() if "pack_blocks_kernel" in n}
    assert len(names) == 2, sorted(names)                    # pack_blocks_kernel and unpack_blocks_kernel
    bad = {n: "REG %d STACK %d LOCAL %d" % u for n, u in names.items() if u[1] or u[2]}
    assert not bad, bad
