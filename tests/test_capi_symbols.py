"""CPU: libb2m.so loads without a GPU and exports every entry point include/b2m.h declares; calls that
need a device fail with an error code, never a crash, and there is no CPU fallback to fall into."""
import ctypes
import os
import re

from marlin_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "b2m.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b2m_[a-z0-9_]+)\s*\(", text)))


def test_every_declared_symbol_is_exported():
    L = _lib.lib()
    names = declared_symbols()
    assert len(names) >= 20
    for n in names:
        assert hasattr(L, n), f"{n} declared in include/b2m.h but not exported by libb2m.so"


def test_version_and_error_paths_without_gpu():
    L = _lib.lib()
    assert b"sm_90a" in L.b2m_version()
    h = ctypes.c_void_p()
    import torch
    if not torch.cuda.is_available():
        rc = L.b2m_ctx_create(0, ctypes.byref(h))
        assert rc == 8  # B2M_ERR_CUDA: no device, and no CPU fallback
        assert L.b2m_last_error()
    assert L.b2m_ntt(None, 0, None, 3, 0, 0) == 1  # B2M_ERR_INVALID_ARG, not a crash


def test_product_does_not_import_the_oracle():
    """The product path must never route through oracle/ (or any CPU fallback)."""
    for dirpath, _, files in os.walk(os.path.join(ROOT, "marlin_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".hpp", ".h")):
                src = open(os.path.join(dirpath, f), errors="ignore").read()
                assert "import oracle" not in src and "from oracle" not in src and "oracle/" not in src, f


def test_header_is_plain_c(tmp_path):
    """include/b2m.h is the drop-in boundary: it must compile as C (no C++-isms, no CUDA / torch types in the signatures)."""
    import subprocess
    src = os.path.join(tmp_path, "use_b2m.c")
    with open(src, "w") as f:
        f.write('#include "b2m.h"\nint main(void) { b2m_rng r; r.kind = B2M_RNG_CALLBACK; r.next_u64 = 0; r.state = 0; (void)r; return B2M_OK; }\n')
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), src])
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "b2m.h")).read(), flags=re.S)  # declarations only
    for banned in ("torch", "at::Tensor", "cudaStream_t", "std::"):
        assert banned not in text, banned


def test_every_declared_symbol_has_a_ctypes_signature_and_a_rust_declaration():
    """The two host-side twins of the header stay complete: marlin_b200/_lib.py sets argtypes for every entry point (an unset
    signature silently truncates 64-bit arguments), and bindings/rust/src/ffi.rs declares the ones the Rust shim binds."""
    L = _lib.lib()
    no_args = {"b2m_last_error", "b2m_version"}
    for n in declared_symbols():
        if n in no_args:
            continue
        assert getattr(L, n).argtypes is not None, f"{n}: no ctypes argtypes in marlin_b200/_lib.py"
    ffi = open(os.path.join(ROOT, "bindings", "rust", "src", "ffi.rs")).read()
    rust_needed = {"b2m_ctx_create", "b2m_ctx_destroy", "b2m_ntt", "b2m_srs_create", "b2m_srs_destroy", "b2m_srs_msm", "b2m_pc_commit", "b2m_pc_open",
                   "b2m_trim", "b2m_ck_destroy", "b2m_ck_commit", "b2m_ck_open_combinations", "b2m_index_create", "b2m_index_destroy",
                   "b2m_index_vk_bytes", "b2m_prove", "b2m_g1_powers", "b2m_fixed_base_msm"}
    assert rust_needed <= set(declared_symbols())
    for n in rust_needed:
        assert re.search(r"pub fn %s\(" % n, ffi), f"{n} missing from bindings/rust/src/ffi.rs"
