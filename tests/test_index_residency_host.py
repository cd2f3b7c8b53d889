"""CPU: the index residency rule of the layout planner (csrc/msm_layout.hpp, msm_plan_residency) and the byte model of a
host-resident index, compiled for the host.  A key plans exactly the device-resident search first and only falls back to an
index that keeps its twelve |K|-vectors in pinned host memory when no device-resident layout fits."""
import ctypes
import os
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
FR = 32


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    src = os.path.join(HERE, "host", "index_residency_host_shim.cpp")
    so = str(tmp_path_factory.mktemp("index_residency") / "libindex_residency.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", src, "-o", so])
    L = ctypes.CDLL(so)
    sz, ci = ctypes.c_size_t, ctypes.c_int
    P = ctypes.POINTER
    L.residency_plan.argtypes = [sz, ci, sz, ci, ci, sz, P(sz)]
    L.residency_plan.restype = None
    L.residency_search.argtypes = [sz, ci, sz, ci, ci, sz, ci, P(sz)]
    L.residency_search.restype = None
    L.residency_bytes.argtypes = [sz, ci, sz, ci, ci, ci, sz, sz, sz, ci, P(sz)]
    L.residency_bytes.restype = None
    return L


KEYS = [  # (n_g, fr_bits, fq_bytes, affine levels, c of the full layout)
    ((1 << 16) + 1, 255, 48, 3, 15), ((1 << 20) * 4, 255, 48, 3, 20), ((1 << 24), 255, 48, 3, 20), ((1 << 26), 255, 48, 3, 20),
    ((1 << 22), 254, 32, 0, 20)]


def plan(L, key, budget):
    n_g, fr_bits, fq, lv, c_full = key
    out = (ctypes.c_size_t * 10)()
    L.residency_plan(n_g, fr_bits, fq, lv, c_full, budget, out)
    return dict(zip(("c", "W", "T", "cap", "tables", "circuit", "msm", "total", "host_index", "host"), list(out)))


def search(L, key, budget, host):
    n_g, fr_bits, fq, lv, c_full = key
    out = (ctypes.c_size_t * 5)()
    L.residency_search(n_g, fr_bits, fq, lv, c_full, budget, int(host), out)
    return dict(zip(("c", "W", "T", "cap", "total"), list(out)))


def model(L, key, c, T, cap, K, H, host):
    n_g, fr_bits, fq, lv, _ = key
    out = (ctypes.c_size_t * 5)()
    L.residency_bytes(n_g, fr_bits, fq, lv, c, T, cap, K, H, int(host), out)
    return dict(zip(("tables", "circuit", "msm", "total", "host"), list(out)))


@pytest.mark.parametrize("key", KEYS, ids=lambda k: f"n{k[0]}_fq{k[2]}")
def test_device_residency_whenever_a_device_layout_fits(lib, key):
    """Over budgets from far too small to everything: the plan is the device search's whenever that finds a layout, and the
    host-resident search's only when it does not; what the plan picks never exceeds the budget."""
    full = search(lib, key, 1 << 62, False)["total"]
    seen_host = False
    for k in range(1, 97):
        budget = full * k // 64
        p = plan(lib, key, budget)
        dev = search(lib, key, budget, False)
        if dev["T"]:
            assert p["host_index"] == 0 and (p["c"], p["T"], p["cap"], p["total"]) == (dev["c"], dev["T"], dev["cap"], dev["total"])
        else:
            host = search(lib, key, budget, True)
            assert p["T"] == host["T"]
            if host["T"]:
                seen_host = True
                assert p["host_index"] == 1 and p["total"] == host["total"]
        if p["T"]:
            assert p["total"] <= budget
    assert seen_host, "some budget fits only a host-resident index"


@pytest.mark.parametrize("log_k,log_h", [(12, 10), (16, 14), (20, 18), (26, 24), (20, 20), (14, 18)])
def test_host_term_drops_the_twelve_vectors_at_rest_but_not_at_build(lib, log_k, log_h):
    """The host-resident circuit term is the larger of the build (twelve vectors on the device) and the proof without them;
    it never exceeds the device-resident term, and pins exactly 12 |K| Fr."""
    key = KEYS[3]
    K, H = 1 << log_k, 1 << log_h
    d = model(lib, key, 16, 4, 1 << 20, K, H, False)
    h = model(lib, key, 16, 4, 1 << 20, K, H, True)
    assert h["host"] == 12 * K * FR and d["host"] == 0
    assert h["circuit"] <= d["circuit"] + 6 * min(K, 1 << 20) * FR  # (the stager's two slots of three vectors)
    assert h["circuit"] >= d["circuit"] - 12 * K * FR
    assert (d["tables"], d["msm"]) == (h["tables"], h["msm"])


def test_2p26_powers_under_an_h100_budget_plan_a_host_resident_index(lib):
    """2^26 powers (2^24 constraints, |K| = 2^26) under 84.46 GB: no device-resident layout fits, a host-resident one does."""
    key = ((1 << 26), 255, 48, 3, 20)
    budget = int(84.46e9)
    assert search(lib, key, budget, False)["T"] == 0
    p = plan(lib, key, budget)
    assert p["T"] >= 1 and p["host_index"] == 1 and p["total"] <= budget
    assert p["host"] == 12 * (1 << 26) * FR


def test_prover_term_is_the_largest_phase(lib):
    """The prover term is a maximum over its phases, not their sum: at |K| = 4|H| it grows with |K| like round 3 (13 |K|) and
    at |K| << |H| like rounds 1-2 (42 |H|)."""
    key = KEYS[3]
    H = 1 << 20
    a = model(lib, key, 16, 4, 1 << 20, 4 * H, H, False)["circuit"]
    b = model(lib, key, 16, 4, 1 << 20, 8 * H, H, False)["circuit"]
    # from |K| = 4H to 8H: the twelve vectors (12), the index structures (2 (4 + 32) + 3 * 37 + 32 bytes) and round 3 (13)
    per_k = 12 * FR + 2 * 36 + 3 * 37 + 32 + 13 * FR
    assert b - a == 4 * H * per_k
