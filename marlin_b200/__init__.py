"""marlin_b200 -- H100-native (sm_90a) Marlin prover hot path.

Host-side mirror of the reference's public API for this path
(`Marlin::<F, PC, FS>::{index, prove}` [reference src/lib.rs:100-311]) over the C ABI in
include/b2m.h.  All arithmetic runs in hand-written CUDA inside libb2m.so; there is no CPU
fallback -- importing `marlin_b200.api` without the built library raises.
"""
from . import _lib  # noqa: F401

__all__ = ["_lib"]
