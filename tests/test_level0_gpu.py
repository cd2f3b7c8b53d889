"""GPU parity tests for the Level-0 ABI (b2m_ntt, b2m_srs_msm, b2m_g1_powers) against the oracle.

Bit-exact bar: NTT vectors equal the oracle's element for element; MSM results equal the
oracle's affine point (unique representation)."""
import ctypes
import random

import numpy as np
import pytest

from marlin_b200 import _lib
from oracle import ec
from oracle.params import BLS12_381, BN254
from oracle.poly import Domain
import b2m_testutil as util

pytestmark = pytest.mark.gpu

CURVES = [BLS12_381, BN254]


@pytest.mark.parametrize("curve", CURVES, ids=lambda c: c.name)
@pytest.mark.parametrize("log_n", [0, 1, 2, 3, 4, 7, 8, 9, 10, 13, 16])
def test_ntt_matches_oracle(b2m_ctx, curve, log_n):
    L = _lib.lib()
    rnd = random.Random(100 + log_n)
    f = curve.fr
    n = 1 << log_n
    vals = [rnd.randrange(f.p) for _ in range(n)]
    vals[0] = 0
    vals[-1] = f.p - 1
    d = Domain(f, n)
    for inverse, coset in ((0, 0), (1, 0), (0, 1), (1, 1)):
        buf = util.fr_to_mont_limbs(curve, vals)
        _lib.check(L.b2m_ntt(b2m_ctx, util.CURVE_ID[curve.name], _lib.ptr(buf), log_n, inverse, coset))
        got = util.fr_from_mont_limbs(curve, buf)
        want = {(0, 0): d.fft, (1, 0): d.ifft, (0, 1): d.coset_fft, (1, 1): d.coset_ifft}[(inverse, coset)](vals)
        assert got == want, (curve.name, log_n, inverse, coset)


@pytest.mark.parametrize("log_n", [20, 22])
def test_ntt_large_roundtrip_and_point_check(b2m_ctx, log_n):
    """Full-size property checks: ifft(fft(x)) == x and evals[k] == p(w^k) at a few k (Horner in Python)."""
    L = _lib.lib()
    curve = BLS12_381
    f = curve.fr
    n = 1 << log_n
    rng = np.random.default_rng(log_n)
    # random canonical values < 2^252 < r, marshalled as "Montgomery limbs" directly: the transform is
    # linear, so any field elements do; keep the python-side decode cheap by checking few positions.
    buf = rng.integers(0, 1 << 63, size=(n, 4), dtype=np.uint64)
    buf[:, 3] &= np.uint64((1 << 60) - 1)
    orig = buf.copy()
    _lib.check(L.b2m_ntt(b2m_ctx, 0, _lib.ptr(buf), log_n, 0, 0))
    d = Domain(f, n)
    _lib.check(L.b2m_ntt(b2m_ctx, 0, _lib.ptr(buf), log_n, 1, 0))
    assert np.array_equal(buf, orig)
    # point check on a sparse polynomial: x has only 3 non-zero coefficients
    sp = np.zeros((n, 4), dtype=np.uint64)
    idx = [0, 5, n - 1]
    cv = [7, 11, 13]
    for i, c in zip(idx, cv):
        sp[i] = _lib.ints_to_limbs([f.to_mont(c)], 4)[0]
    _lib.check(L.b2m_ntt(b2m_ctx, 0, _lib.ptr(sp), log_n, 0, 0))
    for k in (0, 1, 2, n // 2, n // 2 + 3, n - 1, 12345 % n):
        w = d.element(k)
        want = sum(c * pow(w, i, f.p) for i, c in zip(idx, cv)) % f.p
        assert f.from_mont(_lib.limbs_to_ints(sp[k])[0]) == want


@pytest.mark.parametrize("curve", CURVES, ids=lambda c: c.name)
def test_g1_powers_matches_oracle(b2m_ctx, curve):
    beta = 0x1234567890abcdef1234567890abcdef % curve.fr.p
    got = util.points_from_limbs(curve, util.gpu_powers(b2m_ctx, curve, curve.g, beta, 40))
    want = ec.fixed_base_powers(curve, curve.g, beta, 40)
    assert got == want


@pytest.mark.parametrize("curve", CURVES, ids=lambda c: c.name)
def test_fixed_base_msm_matches_oracle(b2m_ctx, curve):
    """b2m_fixed_base_msm (`FixedBaseMSM::multi_scalar_mul` of KZG10::setup): scalars with zero bytes / zero / r - 1 / one, a base
    other than the generator, and more points than one normalisation batch; and b2m_g1_powers across a batch boundary."""
    import ctypes
    rnd = random.Random(77)
    r = curve.fr.p
    base = ec.scalar_mul(curve, 0xabcdef12345, curve.g)
    sc = [0, 1, 2, r - 1, 1 << 200, (1 << 64) + 255, 0xff00ff00ff00] + [rnd.randrange(r) for _ in range(30)]
    out = np.zeros((len(sc), 2 * curve.fq.limbs64), dtype=np.uint64)
    _lib.check(_lib.lib().b2m_fixed_base_msm(b2m_ctx, util.CURVE_ID[curve.name], _lib.ptr(util.points_to_limbs(curve, [base])),
                                             _lib.ptr(util.fr_to_canon_limbs(curve, sc)), len(sc), _lib.ptr(out)))
    assert util.points_from_limbs(curve, out) == [ec.scalar_mul(curve, k, base) if k else None for k in sc]
    beta = 0x5eed5eed5eed5eed5eed5eed % r
    n = 1000
    got = util.points_from_limbs(curve, util.gpu_powers(b2m_ctx, curve, curve.g, beta, n))
    for i in (0, 1, 15, 16, 17, 255, 256, 999):
        assert got[i] == ec.scalar_mul(curve, pow(beta, i, r), curve.g), i


@pytest.mark.parametrize("curve", CURVES, ids=lambda c: c.name)
@pytest.mark.parametrize("window_bits", [0, 8, 11])
def test_msm_small_sizes_match_oracle(b2m_ctx, curve, window_bits):
    rnd = random.Random(7)
    r = curve.fr.p
    beta = rnd.randrange(1, r)
    N = 600
    powers = util.gpu_powers(b2m_ctx, curve, curve.g, beta, N)
    pts = util.points_from_limbs(curve, powers)
    srs = util.make_srs(b2m_ctx, curve, powers, window_bits=window_bits)
    try:
        for n, off in ((0, 0), (1, 0), (2, 5), (3, 0), (31, 1), (32, 0), (100, 17), (513, 87), (600, 0)):
            sc = [rnd.randrange(r) for _ in range(n)]
            if n >= 3:
                sc[0], sc[1], sc[2] = 0, 1, r - 1
            got = util.srs_msm(srs, curve, off, sc)
            want = ec.msm_pippenger_arkworks(curve, pts[off:off + n], sc)
            assert got == want, (n, off)
            assert got == util.trapdoor_msm(curve, curve.g, beta, off, sc)
        # degenerate inputs: all zero, all one, all r-1, all equal
        for sc in ([0] * 64, [1] * 64, [r - 1] * 64, [rnd.randrange(r)] * 64):
            assert util.srs_msm(srs, curve, 3, sc) == util.trapdoor_msm(curve, curve.g, beta, 3, sc)
        # slice past the end is rejected with the reference's degree error, not a crash
        with pytest.raises(_lib.B2MError) as ei:
            util.srs_msm(srs, curve, N - 3, [1, 2, 3, 4])
        assert ei.value.code == 6
    finally:
        _lib.lib().b2m_srs_destroy(srs)


def test_msm_duplicate_and_opposite_bases(b2m_ctx):
    """Bases that collide inside one bucket (P, P, -P): exercises the doubling / cancellation branches."""
    curve = BLS12_381
    rnd = random.Random(11)
    r = curve.fr.p
    P = ec.scalar_mul(curve, 5, curve.g)
    Q = ec.scalar_mul(curve, 9, curve.g)
    pts = [P, P, ec.affine_neg(curve, P), Q, P, None, Q, ec.affine_neg(curve, Q)] * 8
    limbs = util.points_to_limbs(curve, pts)
    srs = util.make_srs(b2m_ctx, curve, limbs, window_bits=8)
    try:
        for trial in range(6):
            sc = [rnd.randrange(r) for _ in pts] if trial else [3] * len(pts)
            assert util.srs_msm(srs, curve, 0, sc) == ec.msm_naive(curve, pts, sc)
    finally:
        _lib.lib().b2m_srs_destroy(srs)


def test_msm_one_shot_abi(b2m_ctx):
    curve = BLS12_381
    L = _lib.lib()
    rnd = random.Random(5)
    pts = [ec.scalar_mul(curve, rnd.randrange(1, curve.fr.p), curve.g) for _ in range(20)]
    sc = [rnd.randrange(curve.fr.p) for _ in pts]
    out = np.zeros(12, dtype=np.uint64)
    inf = ctypes.c_int(0)
    _lib.check(L.b2m_msm_g1(b2m_ctx, 0, _lib.ptr(util.points_to_limbs(curve, pts)), _lib.ptr(util.fr_to_canon_limbs(curve, sc)),
                            len(pts), _lib.ptr(out), ctypes.byref(inf)))
    assert util.points_from_limbs(curve, out)[0] == ec.msm_naive(curve, pts, sc)


@pytest.mark.parametrize("log_n", [16, 20])
def test_msm_large_trapdoor(b2m_ctx, log_n):
    """Full-size check that needs no slow oracle: bases are beta^i*g, so the MSM must equal
    (sum s_i beta^i) * g.  Random scalars, plus a slice at a non-zero offset."""
    curve = BLS12_381
    r = curve.fr.p
    n = 1 << log_n
    beta = 0x2f8a9b1c3d4e5f60718293a4b5c6d7e8f9 % r
    powers = util.gpu_powers(b2m_ctx, curve, curve.g, beta, n)
    srs = util.make_srs(b2m_ctx, curve, powers)
    try:
        rng = np.random.default_rng(3)
        raw = rng.integers(0, 1 << 63, size=(n, 4), dtype=np.uint64)
        raw[:, 3] &= np.uint64((1 << 61) - 1)  # < 2^253 < r
        sc = _lib.limbs_to_ints(raw)
        assert util.srs_msm(srs, curve, 0, sc) == util.trapdoor_msm(curve, curve.g, beta, 0, sc)
        m = n // 2 + 1
        assert util.srs_msm(srs, curve, 77, sc[:m]) == util.trapdoor_msm(curve, curve.g, beta, 77, sc[:m])
    finally:
        _lib.lib().b2m_srs_destroy(srs)


def test_msm_skewed_scalars(b2m_ctx):
    """Scalar distributions that put most references in a handful of buckets (a polynomial whose
    coefficients are nearly all equal, as z_A of the reference's DummyCircuit is): exercises the
    cut-bucket stitching, including the long-run path."""
    curve = BLS12_381
    r = curve.fr.p
    n = 1 << 16
    beta = 0x1b2c3d4e5f60718293a4b5c6d7e8f9 % r
    powers = util.gpu_powers(b2m_ctx, curve, curve.g, beta, n)
    srs = util.make_srs(b2m_ctx, curve, powers)
    rnd = random.Random(21)
    try:
        v, w = rnd.randrange(r), rnd.randrange(r)
        cases = [[v] * n, [v if i % 3 else w for i in range(n)], [v] * (n - 5) + [rnd.randrange(r) for _ in range(5)],
                 [(i % 7) + 1 for i in range(n)], [r - 1 - (i % 2) for i in range(n)]]
        for sc in cases:
            assert util.srs_msm(srs, curve, 0, sc) == util.trapdoor_msm(curve, curve.g, beta, 0, sc)
    finally:
        _lib.lib().b2m_srs_destroy(srs)


@pytest.mark.gpu
@pytest.mark.parametrize("levels,T,variant,upper,mapping", [
    (1, 1, 4, 4, 1), (2, 3, 4, 4, 1), (3, 64, 4, 4, 1), (4, 5, 3, 3, 1), (6, 2, 5, 5, 1),   # fused kernel variants, default (interleaved) mapping
    (3, 64, 8, 8, 1), (2, 3, 9, 9, 1), (4, 1, 9, 8, 0), (1, 7, 8, 8, 1),                    # software-pipelined kernels
    (3, 64, 11, 13, 1), (2, 3, 12, 11, 1), (4, 1, 13, 12, 0), (3, 5, 13, 11, 1), (1, 64, 12, 12, 1),  # split: two kernels per level
    (3, 64, 21, 21, 1), (2, 3, 22, 21, 1), (4, 1, 21, 22, 0), (3, 16, 22, 22, 1), (1, 5, 21, 21, 1),          # split + level-wide batch inversion
    (3, 64, 4, 4, 0), (2, 5, 3, 5, 0)])                                                     # blocked mapping
def test_msm_affine_levels_forced(b2m_ctx, monkeypatch, levels, T, variant, upper, mapping):
    """The batched-affine levels (csrc/msm_affine.cuh) are skipped for small MSMs; force them on (any size, odd
    batch lengths, every kernel variant) over the inputs that hit their special cases: colliding bases (P + P,
    P - P inside a bucket, at level 0 and above), zero / equal / tiny scalars, buckets of every parity."""
    monkeypatch.setenv("B2M_MSM_AFFINE_LEVELS", str(levels))
    monkeypatch.setenv("B2M_MSM_AFFINE_T", str(T))
    monkeypatch.setenv("B2M_MSM_AFFINE_CTAS", str(variant))
    monkeypatch.setenv("B2M_MSM_AFFINE_CTAS_UPPER", str(upper))
    monkeypatch.setenv("B2M_MSM_AFFINE_MAP", str(mapping))
    monkeypatch.setenv("B2M_MSM_AFFINE_MIN_REFS", "0")
    curve = BLS12_381
    r = curve.fr.p
    rnd = random.Random(31 + levels)
    P = ec.scalar_mul(curve, 5, curve.g)
    Q = ec.scalar_mul(curve, 9, curve.g)
    pts = [P, P, ec.affine_neg(curve, P), Q, P, None, Q, ec.affine_neg(curve, Q)] * 8
    srs = util.make_srs(b2m_ctx, curve, util.points_to_limbs(curve, pts), window_bits=8)
    try:
        for trial in range(4):
            sc = [rnd.randrange(r) for _ in pts] if trial else [3] * len(pts)
            assert util.srs_msm(srs, curve, 0, sc) == ec.msm_naive(curve, pts, sc)
    finally:
        _lib.lib().b2m_srs_destroy(srs)
    n = 1 << 12
    beta = 3  # tiny beta: beta^i * g collide with the 2^(c w) multiples of the window tables
    powers = util.gpu_powers(b2m_ctx, curve, curve.g, beta, n)
    for wb in (8, 0):
        srs = util.make_srs(b2m_ctx, curve, powers, window_bits=wb)
        try:
            v, w = rnd.randrange(r), rnd.randrange(r)
            cases = [[v] * n, [v if i % 3 else w for i in range(n)], [(i % 7) + 1 for i in range(n)], [r - 1 - (i % 2) for i in range(n)],
                     [rnd.randrange(r) for _ in range(n)], [0] * n, [1] * 5, [rnd.randrange(r) for _ in range(777)]]
            for sc in cases:
                assert util.srs_msm(srs, curve, 1, sc[:n - 1]) == util.trapdoor_msm(curve, curve.g, beta, 1, sc[:n - 1])
        finally:
            _lib.lib().b2m_srs_destroy(srs)
