"""CPU: the reduced-table MSM layout (csrc/msm_layout.hpp, csrc/msm_impl.cuh).

A key that keeps T < W window tables reads window w from table w // m (m = ceil(W / T), table j = 2^(c m j) P) and sends its
digit to bucket set w % m; the sets are reduced separately and recombined by Horner as sum_k 2^(c k) S_k.  A Python-integer
mirror of that digit -> (table, set, bucket) map and of the recombination reconstructs every scalar for every width
8 <= c <= 24 and table count, on edge scalars.  The layout planner and its byte model are compiled for the host and checked
for the rules the library relies on: all tables whenever they fit, T monotone in the budget, the 24-bit bucket field."""
import ctypes
import os
import random
import subprocess

import pytest

from oracle.params import BLS12_381, BN254

HERE = os.path.dirname(os.path.abspath(__file__))
BKT_BITS = 24
FR_BITS = {"bls12_381": 255, "bn254": 254}  # Fr::Params::BITS
CURVES = [BLS12_381, BN254]


def windows(fr_bits, c):
    return (fr_bits + 1 + c - 1) // c


def digits(s, c, W):
    """msm_digits_kernel: signed c-bit digits of a canonical scalar (256-bit limbs), lowest window first."""
    half, carry, out = 1 << (c - 1), 0, []
    for w in range(W):
        raw = (s >> (w * c)) & ((1 << c) - 1) if w * c < 256 else 0
        v = raw + carry
        if v > half:
            out.append(v - (1 << c))
            carry = 1
        else:
            out.append(v)
            carry = 0
    assert carry == 0, "the top window leaves no carry"
    return out


NO_DIGIT = 0xFFFFFFFF


def encode(d, w, m, c):
    """msm_digits_kernel's word for digit d of window w: (set offset + |d| - 1) | sign << 31, NO_DIGIT for d = 0 -- including
    the zero digit left by an all-ones window plus a carry, which must not wrap into the previous set's last bucket."""
    if d == 0:
        return NO_DIGIT
    return ((w % m) * (1 << (c - 1)) + abs(d) - 1) | (0x80000000 if d < 0 else 0)


def references(s, c, W, T):
    """(table, bucket id, sign) per non-zero digit, as msm_scatter_kernel sorts them."""
    m = -(-W // T)
    B = 1 << (c - 1)
    refs = []
    for w, d in enumerate(digits(s, c, W)):
        word = encode(d, w, m, c)
        if word != NO_DIGIT:
            refs.append((w // m, word & 0x7FFFFFFF, -1 if word >> 31 else 1))
    return refs, m, B


def recombine(refs, c, m, B):
    """Bucket sums on integer 'points' (table j holds 2^(c m j)), per-set sum_b (b + 1) B_b, then Horner over the sets."""
    buckets = {}
    for j, bkt, sign in refs:
        buckets[bkt] = buckets.get(bkt, 0) + sign * (1 << (c * m * j))
    sets = [sum((b - k * B + 1) * v for b, v in buckets.items() if b // B == k) for k in range(m)]
    acc = sets[m - 1]
    for k in range(m - 2, -1, -1):
        acc = (acc << c) + sets[k]
    return acc


def edge_scalars(r, c, rnd):
    half = 1 << (c - 1)
    out = [0, 1, 2, r - 1, r - 2, half, half + 1, (1 << c) - 1, 1 << 200, (1 << 254) - 1 if (1 << 254) - 1 < r else r - 3]
    # all-carry patterns: every window half + 1 (a negative digit and a carry into the next), or all ones
    for pat in (half + 1, (1 << c) - 1, half):
        v = 0
        for w in range(0, 256, c):
            v |= pat << w
        out.append(v % r)
    return out + [rnd.randrange(r) for _ in range(4)]


@pytest.mark.parametrize("curve", CURVES, ids=lambda cv: cv.name)
@pytest.mark.parametrize("c", range(8, 25))
def test_digit_map_and_horner_reconstruct_the_scalar(curve, c):
    rnd = random.Random(c)
    r = curve.fr.p
    W = windows(FR_BITS[curve.name], c)
    Ts = sorted({1, 2, 3, W - 1, W, max(1, W // 2), max(1, W // 3 + 1)} - {0})
    assert any(W % T for T in Ts), "W not a multiple of T is covered"
    for T in Ts:
        m = -(-W // T)
        if (m << (c - 1)) > (1 << BKT_BITS):
            continue  # the library refuses this layout (msm_sets_fit)
        for s in edge_scalars(r, c, rnd):
            refs, m, B = references(s, c, W, T)
            for j, bkt, _ in refs:
                assert 0 <= j < T and j < 256, "table index fits the 8-bit field of a sorted reference"
                assert 0 <= bkt < m * B <= 1 << BKT_BITS
            assert recombine(refs, c, m, B) == s, (c, T, s)


@pytest.fixture(scope="module")
def hostlib(tmp_path_factory):
    src = os.path.join(HERE, "host", "msm_layout_host_shim.cpp")
    so = str(tmp_path_factory.mktemp("msm_layout") / "libmsm_layout.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", src, "-o", so])
    L = ctypes.CDLL(so)
    sz, ci = ctypes.c_size_t, ctypes.c_int
    P = ctypes.POINTER
    L.layout_plan.argtypes = [sz, sz, ci, sz, ci, ci, ci, ci, sz, ci, sz, P(sz)]
    L.layout_plan.restype = None
    L.layout_bytes.argtypes = [sz, sz, ci, sz, ci, ci, ci, sz, P(sz)]
    L.layout_bytes.restype = None
    L.layout_sets_fit.argtypes = [ci, ci]
    return L


KEYS = [  # (n_g, fr_bits, fq_bytes, affine levels, c of the full layout)
    ((1 << 16) + 1, 255, 48, 3, 15), ((1 << 20) * 4, 255, 48, 3, 20), ((1 << 25), 255, 48, 3, 20), ((1 << 26), 255, 48, 3, 20),
    ((1 << 22), 254, 32, 0, 20)]


def plan(L, key, budget, forced_T=0, forced_cap=0):
    n_g, fr_bits, fq, lv, c_full = key
    out = (ctypes.c_size_t * 8)()
    L.layout_plan(n_g, 3, fr_bits, fq, lv, c_full, min(c_full, 16), 8, budget, forced_T, forced_cap, out)
    return dict(zip(("c", "W", "T", "cap", "tables", "circuit", "msm", "total"), list(out)))


def model(L, key, c, T, cap):
    n_g, fr_bits, fq, lv, _ = key
    out = (ctypes.c_size_t * 4)()
    L.layout_bytes(n_g, 3, fr_bits, fq, lv, c, T, cap, out)
    return list(out)


@pytest.mark.parametrize("key", KEYS, ids=lambda k: f"n{k[0]}_fq{k[2]}")
def test_full_tables_whenever_they_fit(hostlib, key):
    n_g, fr_bits, fq, lv, c_full = key
    W = windows(fr_bits, c_full)
    full = model(hostlib, key, c_full, W, 0)
    assert full[0] == W * (n_g + 3) * 2 * fq
    p = plan(hostlib, key, full[3])
    assert (p["c"], p["T"], p["cap"], p["total"]) == (c_full, W, 0, full[3])
    p = plan(hostlib, key, 1 << 60)
    assert (p["T"], p["cap"]) == (W, 0)
    # one byte less: the full tables stay if a pass cap makes them fit, and nothing the plan picks exceeds the budget
    p = plan(hostlib, key, full[3] - 1)
    assert p["T"] == 0 or p["total"] <= full[3] - 1
    if p["T"] and p["c"] == c_full and p["T"] == W:
        assert p["cap"] > 0


@pytest.mark.parametrize("key", KEYS, ids=lambda k: f"n{k[0]}_fq{k[2]}")
def test_tables_monotone_in_the_budget(hostlib, key):
    n_g, fr_bits, fq, lv, c_full = key
    full = model(hostlib, key, c_full, windows(fr_bits, c_full), 0)[3]
    last = None
    for k in range(1, 65):
        budget = full * k // 64
        p = plan(hostlib, key, budget)
        if p["T"]:
            assert p["total"] <= budget
            assert p["total"] == model(hostlib, key, p["c"], p["T"], p["cap"])[3]
            mm = -(-p["W"] // p["T"])
            assert hostlib.layout_sets_fit(p["c"], mm) and (mm << (p["c"] - 1)) <= 1 << BKT_BITS
            assert p["T"] == -(-p["W"] // mm), "every table kept is read by some window"
        # tables kept (bytes of them) never shrink when the budget grows
        tb = p["tables"] if p["T"] else 0
        if last is not None:
            assert tb >= last, (k, p)
        last = tb
    assert plan(hostlib, key, full)["T"] == windows(fr_bits, c_full)
    # below the smallest layout nothing fits, and the figures reported are that layout's
    tiny = plan(hostlib, key, 1 << 20)
    assert tiny["T"] == 0 and tiny["total"] > 1 << 20


def test_bucket_field_limits_the_sets(hostlib):
    """m 2^(c-1) <= 2^24: at c = 24 a key can drop to ceil(W / 2) tables but no further; forcing fewer is refused."""
    key = ((1 << 20), 255, 48, 3, 24)
    W = windows(255, 24)
    for T in range(1, W + 1):
        m = -(-W // T)
        assert bool(hostlib.layout_sets_fit(24, m)) == ((m << 23) <= 1 << BKT_BITS)
    n_g, fr_bits, fq, lv, _ = key
    out = (ctypes.c_size_t * 8)()
    hostlib.layout_plan(n_g, 3, fr_bits, fq, lv, 24, 24, 24, 1 << 60, 1, 0, out)
    assert out[2] == 0  # T = 1 would need 11 sets of 2^23 buckets
    hostlib.layout_plan(n_g, 3, fr_bits, fq, lv, 24, 24, 24, 1 << 60, (W + 1) // 2, 0, out)
    assert out[2] == (W + 1) // 2


def test_model_shrinks_with_fewer_tables_and_smaller_passes(hostlib):
    key = ((1 << 24), 255, 48, 3, 20)
    c = 16
    W = windows(255, c)
    used = sorted({-(-W // -(-W // T)) for T in range(1, W + 1)})  # the table counts some m reads in full
    by_T = [model(hostlib, key, c, T, 0) for T in used]
    assert all(a[0] < b[0] for a, b in zip(by_T, by_T[1:]))
    by_cap = [model(hostlib, key, c, 1, 1 << lg)[2] for lg in range(16, 23)]
    assert all(a < b for a, b in zip(by_cap, by_cap[1:]))
    assert model(hostlib, key, c, 1, 0)[2] > by_cap[-1]


@pytest.mark.parametrize("W,c", [(16, 16), (13, 20), (32, 8), (24, 11)])
def test_tables_are_normalised_to_the_ones_read(hostlib, W, c):
    """T = 15 at W = 16 gives m = 2 bucket sets, whose windows read tables 0..7 only: the model counts, and a forced layout
    keeps, 8 tables, so the same sets never cost more table bytes (nor a shorter pass) than the T the kernels use."""
    key = ((1 << 20), 255, 48, 3, 20)
    n_g = key[0]
    for T in range(1, W + 1):
        m = -(-W // T)
        used = -(-W // m)
        assert model(hostlib, key, c, T, 0) == model(hostlib, key, c, used, 0)
        assert model(hostlib, key, c, T, 0)[0] == used * (n_g + 3) * 96
        if not hostlib.layout_sets_fit(c, m):
            continue
        out = (ctypes.c_size_t * 8)()
        hostlib.layout_plan(n_g, 3, 255, 48, 3, c, c, c, 1 << 60, T, 0, out)
        assert out[2] == (W if T >= W else used), (T, out[2])
