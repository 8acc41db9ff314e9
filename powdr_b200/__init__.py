"""powdr_b200 -- H100-native STARK proving hot path for powdr autoprecompile (APC) chips over BabyBear.

The product is the sm_90a shared library behind include/powdr_b200.h; this package is the thin host-side mirror of the
reference's Rust call sites (machine JSON -> bytecode, launch wrappers, segment proving).  There is no CPU fallback:
importing works anywhere, but every proving call needs the CUDA library and a GPU.  The verifier (VerifyingKey, verify_chips,
verify_segment, verify_proof_bytes) and the proof's byte form (encode_chips_proof, encode_segment_proof, decode_proof) are host
code in the same library and need no GPU.
"""
from .capi import (Context, Air, Group, VerifyingKey, verify_chips, verify_segment, encode_chips_proof, encode_segment_proof, decode_proof,  # noqa: F401
                   verify_proof_bytes, load_library, LibraryMissing, P)
from .machine import SymbolicMachine, compile_constraints, compile_derived, compile_bus  # noqa: F401

__all__ = ["Context", "Air", "Group", "VerifyingKey", "verify_chips", "verify_segment", "encode_chips_proof", "encode_segment_proof", "decode_proof",
           "verify_proof_bytes", "load_library", "LibraryMissing", "P", "SymbolicMachine", "compile_constraints",
           "compile_derived", "compile_bus"]
