"""GPU: keys with fewer window tables than windows, MSMs split into bounded bucket passes, and the device-memory limit that
chooses between them (csrc/msm_layout.hpp).  An MSM is a unique group element, so every layout must give exactly the
full-table result: MSMs equal (sum s_i beta^i) g, commitments and proofs equal the default key's byte for byte."""
import ctypes
import random

import numpy as np
import pytest

from marlin_b200 import _lib, api
from marlin_b200 import r1cs as gr1cs
from oracle.params import BLS12_381, BN254
import b2m_testutil as util

pytestmark = pytest.mark.gpu

FR_BITS = {"bls12_381": 255, "bn254": 254}


@pytest.fixture
def gctx(b2m_ctx):
    c = api.Context.__new__(api.Context)
    c.handle = b2m_ctx
    return c


def make_srs(ctx, curve, powers, window_bits, window_tables):
    h = ctypes.c_void_p()
    _lib.check(_lib.lib().b2m_srs_create_layout(ctx, util.CURVE_ID[curve.name], _lib.ptr(powers), len(powers), None, None, 0, window_bits,
                                                window_tables, ctypes.byref(h)))
    return h


def check_slices(srs, curve, beta, N, rnd):
    r = curve.fr.p
    cases = [(0, [rnd.randrange(r) for _ in range(N)]),                       # the whole key
             (N // 3, [0, 1, r - 1] + [rnd.randrange(r) for _ in range(997)]),  # the middle
             (N - 500, [rnd.randrange(r) for _ in range(500)]),                # ending at the last power
             (N - 1, [rnd.randrange(r)]), (7, [0] * 300), (0, [r - 1] * 64)]
    for off, sc in cases:
        assert util.srs_msm(srs, curve, off, sc) == util.trapdoor_msm(curve, curve.g, beta, off, sc), (off, len(sc))


@pytest.mark.parametrize("curve", [BLS12_381, BN254], ids=lambda c: c.name)
@pytest.mark.parametrize("c", [8, 11, 16, 20])
def test_reduced_tables_match_trapdoor(b2m_ctx, curve, c):
    W = (FR_BITS[curve.name] + 1 + c - 1) // c
    rnd = random.Random(c)
    beta = rnd.randrange(1, curve.fr.p)
    N = 3000
    powers = util.gpu_powers(b2m_ctx, curve, curve.g, beta, N)
    for T in sorted({1, 2, W - 1, W}):
        srs = make_srs(b2m_ctx, curve, powers, c, T)
        try:
            assert _lib.lib().b2m_srs_window_bits(srs) == c
            m = -(-W // T)
            assert _lib.lib().b2m_srs_window_tables(srs) == -(-W // m)  # only the tables some window reads
            check_slices(srs, curve, beta, N, rnd)
        finally:
            _lib.lib().b2m_srs_destroy(srs)


@pytest.mark.parametrize("c,T", [(8, 1), (11, 2), (16, 1), (16, 15), (20, 1)])
def test_reduced_tables_with_affine_levels_forced(b2m_ctx, monkeypatch, c, T):
    """The batched-affine levels address `tables + table * stride + index` and take the bucket count as a parameter: force them
    on for reduced keys, where one reference's table field is window / m and the buckets are m sets."""
    monkeypatch.setenv("B2M_MSM_AFFINE_LEVELS", "3")
    monkeypatch.setenv("B2M_MSM_AFFINE_MIN_REFS", "0")
    curve = BLS12_381
    rnd = random.Random(100 + c)
    beta = rnd.randrange(1, curve.fr.p)
    N = 3000
    powers = util.gpu_powers(b2m_ctx, curve, curve.g, beta, N)
    srs = make_srs(b2m_ctx, curve, powers, c, T)
    try:
        assert _lib.lib().b2m_srs_affine_levels(srs) == 3
        check_slices(srs, curve, beta, N, rnd)
    finally:
        _lib.lib().b2m_srs_destroy(srs)


@pytest.mark.parametrize("cap", [1000, 4097])
def test_pass_caps(gctx, monkeypatch, cap):
    """2^14-pair MSMs split into passes of `cap` pairs: single MSMs at every slice position, and batches of eight hiding
    commitments (the blinding group rides with the first pass) equal to the uncapped key's."""
    curve = BLS12_381
    n = 1 << 14
    beta = 0x5eed1234 % curve.fr.p
    m = api.Marlin("bls12_381", "marlin_kzg10", ctx=gctx)
    ref = m.srs_from_trapdoor(n + 16, beta=beta)
    monkeypatch.setenv("B2M_MSM_MAX_PAIRS", str(cap))
    capped = m.srs_from_trapdoor(n + 16, beta=beta)
    monkeypatch.delenv("B2M_MSM_MAX_PAIRS")
    try:
        assert capped.layout()["max_pairs"] == cap and ref.layout()["max_pairs"] == 0
        rnd = random.Random(cap)
        r = curve.fr.p
        for off, k in ((0, n), (3, n - 5), (17, cap), (5, cap + 1), (n + 16 - 2 * cap - 1, 2 * cap + 1), (0, 1)):
            sc = [rnd.randrange(r) for _ in range(k)]
            assert util.srs_msm(capped.handle, curve, off, sc) == util.trapdoor_msm(curve, curve.g, beta, off, sc), (off, k)
        rng = np.random.default_rng(cap)
        polys = []
        for i in range(8):
            length = n - 97 * i
            raw = rng.integers(0, 1 << 63, size=(length, 4), dtype=np.uint64)
            raw[:, 3] &= np.uint64((1 << 60) - 1)
            polys.append((raw, None, 1))
        want = m.commit(ref, polys, api.ZkRng(seed=bytes(32)))
        got = m.commit(capped, polys, api.ZkRng(seed=bytes(32)))
        for a, b in zip(want, got):
            assert np.array_equal(a, b)
    finally:
        capped.close()
        ref.close()


def prove_once(m, srs, circ):
    pk = m.index(srs, circ)
    try:
        return pk.vk_bytes, m.prove(pk, circ, api.ZkRng.test_rng()), pk
    except BaseException:
        pk.close()
        raise


@pytest.mark.parametrize("curve_name", ["bls12_381", "bn254"])
@pytest.mark.parametrize("scheme", ["marlin_kzg10", "sonic_kzg10"])
@pytest.mark.parametrize("log_n", [10, 14])
def test_index_and_prove_on_one_table(gctx, monkeypatch, curve_name, scheme, log_n):
    """`index` + `prove` on a key with one window table and 4097-pair MSM passes give the default key's verifier key and proof
    bytes, and the proof verifies on the GPU (and fails for a wrong public input)."""
    n = 1 << log_n
    a, b = 0x1234567890abcdef, 0xfedcba0987654321
    m = api.Marlin(curve_name, scheme, ctx=gctx)
    bounds = (n - 2, 4 * n - 2)
    circ = gr1cs.dummy_circuit(m.curve_id, a, b, 10, n)
    out = []
    for tables, cap in ((0, None), (1, 4097)):
        if cap:
            monkeypatch.setenv("B2M_MSM_MAX_PAIRS", str(cap))
        srs = m.universal_setup(n, n, 3 * n, beta=0x5eed, gamma=7, degree_bounds=bounds, window_tables=tables)
        monkeypatch.delenv("B2M_MSM_MAX_PAIRS", raising=False)
        try:
            lay = srs.layout()
            if tables:
                assert lay["window_tables"] == 1 and lay["max_pairs"] == cap
            vk_bytes, proof, pk = prove_once(m, srs, circ)
            try:
                vk = m.verifier_key(pk, srs)
                try:
                    c_pub = a * b % _lib_modulus(m.curve_id)
                    assert m.verify(vk, [c_pub], proof, api.ZkRng(seed=bytes(32)))
                    assert not m.verify(vk, [(c_pub + 1) % _lib_modulus(m.curve_id)], proof, api.ZkRng(seed=bytes(32)))
                finally:
                    vk.close()
            finally:
                pk.close()
            out.append((vk_bytes, proof))
        finally:
            srs.close()
    assert out[0][0] == out[1][0]
    assert out[0][1] == out[1][1]


def _lib_modulus(cid):
    from marlin_b200 import fields
    return fields.FR_MODULUS[cid]


def test_memory_limit_selects_fewer_tables_and_bounds_the_peak(b2m_ctx):
    """A limit below what a 2^16-power key needs with all its tables: the key keeps fewer, index + prove stay under the limit
    (pool high-water mark) and the proof equals the unlimited key's."""
    n = 1 << 14  # 2^16 powers: |K| = 4 |H| (DummyCircuit with 3n non-zeros)
    a, b = 3, 5
    full_ctx = api.Context(0)
    try:
        m0 = api.Marlin("bls12_381", "marlin_kzg10", ctx=full_ctx)
        circ = gr1cs.dummy_circuit(m0.curve_id, a, b, 10, n)
        srs0 = m0.universal_setup(n, n, 3 * n, beta=0x77, gamma=7)
        try:
            full = srs0.layout()
            assert full["window_tables"] == (256 + full["window_bits"] - 1) // full["window_bits"]
            want_vk, want_proof, pk0 = prove_once(m0, srs0, circ)
            pk0.close()
        finally:
            srs0.close()
    finally:
        full_ctx.close()
    ctx = api.Context(0)
    try:
        m = api.Marlin("bls12_381", "marlin_kzg10", ctx=ctx)
        # (the device pool is shared by every context of the process: the limit counts what is already in use)
        limit = ctx.memory()["used"] + full["model_bytes"] - full["tables_bytes"] // 2
        _lib.check(_lib.lib().b2m_ctx_set_memory_limit(ctx.handle, limit))
        srs = m.universal_setup(n, n, 3 * n, beta=0x77, gamma=7)
        try:
            lay = srs.layout()
            assert 1 <= lay["window_tables"] < full["window_tables"]
            assert lay["model_bytes"] <= lay["budget"] <= limit
            vk_bytes, proof, pk = prove_once(m, srs, circ)
            pk.close()
            peak = ctx.memory()["peak"]
            assert peak <= limit, (peak, limit, lay)
            assert (vk_bytes, proof) == (want_vk, want_proof)
        finally:
            srs.close()
    finally:
        ctx.close()


def test_forced_tables_beyond_the_bucket_field_are_an_invalid_argument(b2m_ctx):
    """c = 24 has 11 windows; one table would need 11 sets of 2^23 buckets, more than the 24-bit bucket field holds."""
    curve = BLS12_381
    powers = util.gpu_powers(b2m_ctx, curve, curve.g, 5, 64)
    with pytest.raises(_lib.B2MError) as ei:
        make_srs(b2m_ctx, curve, powers, 24, 1)
    assert ei.value.code == 1 and "bucket" in str(ei.value)
    srs = make_srs(b2m_ctx, curve, powers, 24, 6)  # 2 sets: fits
    try:
        assert _lib.lib().b2m_srs_window_tables(srs) == 6
    finally:
        _lib.lib().b2m_srs_destroy(srs)


def test_memory_limit_below_the_minimum_is_a_clean_error(b2m_ctx):
    n = 1 << 12
    ctx = api.Context(0, memory_limit=1 << 20)
    try:
        m = api.Marlin("bls12_381", "marlin_kzg10", ctx=ctx)
        with pytest.raises(_lib.B2MError) as ei:
            m.universal_setup(n, n, 3 * n, beta=0x77, gamma=7)
        assert ei.value.code == _lib.ERR_MEMORY_LIMIT
        assert "bytes" in str(ei.value) and "budget" in str(ei.value)
        # a key made under a generous limit, then an index after the limit was lowered: refused before allocating
        _lib.check(_lib.lib().b2m_ctx_set_memory_limit(ctx.handle, 0))
        srs = m.universal_setup(n, n, 3 * n, beta=0x77, gamma=7)
        try:
            _lib.check(_lib.lib().b2m_ctx_set_memory_limit(ctx.handle, ctx.memory()["used"] + (1 << 20)))
            with pytest.raises(_lib.B2MError) as ei:
                m.index(srs, gr1cs.dummy_circuit(m.curve_id, 3, 5, 10, n))
            assert ei.value.code == _lib.ERR_MEMORY_LIMIT
        finally:
            srs.close()
    finally:
        ctx.close()
