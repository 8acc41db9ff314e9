"""CPU checks of the library's group (pb_group_create, pb_prove_chips_group, pb_query_chips_group): argument checks that need no device,
and examples/group_demo.c, a plain C client that needs nothing but the header and the .so."""
import ctypes as C
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_null_arguments_and_world_are_refused_without_a_device():
    from powdr_b200.capi import Chip, ChipsProof, load_library
    lib = load_library()
    out = C.c_void_p()
    ctxs = (C.c_void_p * 16)()                                     # NULL contexts: never read when the world is wrong
    assert lib.pb_group_create(None, C.c_int(2), C.byref(out)) == -1
    assert lib.pb_group_create(ctxs, C.c_int(2), None) == -1
    for world in (0, 1, 3, 5, 6, 12, 32, -2):
        assert lib.pb_group_create(ctxs, C.c_int(world), C.byref(out)) == -2, world
    assert lib.pb_group_create(ctxs, C.c_int(4), C.byref(out)) == -1          # NULL contexts in a valid world
    assert lib.pb_group_destroy(None) == 0
    arr = (Chip * 1)(Chip(None, None, 8, 4))
    rows = (C.c_void_p * 2)(C.addressof(arr), C.addressof(arr))
    proof, cs = ChipsProof(), (C.c_uint32 * 4)()
    assert lib.pb_prove_chips_group(None, rows, C.c_size_t(1), C.byref(proof), cs) == -1
    assert lib.pb_query_chips_group(None, None, C.c_size_t(0), None, C.c_size_t(0)) == -1


def test_group_demo_links_and_fails_loudly_without_a_gpu(tmp_path):
    """examples/group_demo.c compiles as plain C99 against the header; without a device it exits with PB_ERR_NO_DEVICE, like abi_demo"""
    import powdr_b200
    powdr_b200.load_library()
    exe = str(tmp_path / "group_demo")
    lib_dir = os.path.join(ROOT, "powdr_b200", "_lib")
    subprocess.check_call(["/usr/bin/gcc", "-std=c99", "-O2", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "examples", "group_demo.c"), "-L", lib_dir, "-lpowdr_b200", "-Wl,-rpath," + lib_dir, "-o", exe])
    r = subprocess.run([exe, "9"], capture_output=True, text=True, timeout=600)
    if r.returncode != 0:
        assert "pb_ctx_create" in r.stderr and "-> -5" in r.stderr, r.stderr
    else:                                   # a GPU is present where this CPU suite runs: the demo must then prove and verify
        assert "verify 0" in r.stdout, r.stdout
