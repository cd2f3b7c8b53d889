"""GPU: NTTs and MSMs at the sizes a 2^24-constraint proof runs, exact against the CPU reference.

NTTs of 2^17 to 2^27 points take three and four passes of the transform (NTT_MAX_K = 8 stages per pass); they are compared
limb for limb with oracle/cport (ark-poly's radix-2 FFT) in all four (inverse, coset) modes.  MSMs reach the XYZZ-only bucket
pass at millions of points, the overflow of the stitch queues, every window width from 17 to 24 and the one-shot
`b2m_msm_g1` path; they are checked against the trapdoor (bases beta^i g) or against cport's Pippenger.

Every comparison is of raw uint64 limbs, and every GPU output is checked to be fully reduced (below its modulus): an output
of x + p would pass a comparison through `from_mont`, but not the prover's bit-for-bit comparisons of field elements."""
import ctypes

import numpy as np
import pytest

import b2m_testutil as util
from marlin_b200 import _lib
from oracle import cport, ec
from oracle.params import BLS12_381, BN254
from oracle.poly import Domain

pytestmark = pytest.mark.gpu

CURVES = [BLS12_381, BN254]
ERR_DEGREE_TOO_LARGE = 6
LONG_CAP = 1 << 18   # entries of each stitch queue (msm_impl.cuh, run_pass)
Q_BOUND = 80         # references per accumulate thread: the launch picks q near MSM_Q = 64 at these sizes


def _mem_available():
    try:
        with open("/proc/meminfo") as fh:
            for line in fh:
                if line.startswith("MemAvailable:"):
                    return int(line.split()[1]) * 1024
    except OSError:
        pass
    return 0


def _require_memory(gpu_bytes, host_bytes):
    import torch
    total = torch.cuda.get_device_properties(0).total_memory
    avail = _mem_available()
    if total < gpu_bytes or avail < host_bytes:
        pytest.skip(f"needs a GPU of >= {gpu_bytes / 1e9:.0f} GB (has {total / 1e9:.1f} GB) and >= {host_bytes / 2**30:.0f} GiB "
                    f"MemAvailable (has {avail / 2**30:.1f} GiB)")


def _modulus_limbs(p, nlimbs):
    return np.array([(p >> (64 * j)) & ((1 << 64) - 1) for j in range(nlimbs)], dtype=np.uint64)


def below(arr, p):
    """Per row of little-endian uint64 limbs: value < p (vectorised lexicographic compare from the top limb)."""
    arr = np.asarray(arr, dtype=np.uint64).reshape(-1, (p.bit_length() + 63) // 64)
    pl = _modulus_limbs(p, arr.shape[1])
    lt = np.zeros(len(arr), dtype=bool)
    eq = np.ones(len(arr), dtype=bool)
    for j in range(arr.shape[1] - 1, -1, -1):
        lt |= eq & (arr[:, j] < pl[j])
        eq &= arr[:, j] == pl[j]
    return lt


def uniform_below(rng, n, p):
    """(n, limbs) uint64 uniform in [0, p) (rejection sampling on the top limb's bit length)."""
    nl = (p.bit_length() + 63) // 64
    top_mask = np.uint64((1 << (p.bit_length() - 64 * (nl - 1))) - 1)
    out = rng.integers(0, 1 << 64, size=(n, nl), dtype=np.uint64, endpoint=False)
    out[:, -1] &= top_mask
    bad = ~below(out, p)
    while bad.any():
        k = int(bad.sum())
        fresh = rng.integers(0, 1 << 64, size=(k, nl), dtype=np.uint64, endpoint=False)
        fresh[:, -1] &= top_mask
        out[bad] = fresh
        bad = ~below(out, p)
    return out


def limbs_to_ints(arr):
    b = np.ascontiguousarray(arr, dtype="<u8").tobytes()
    w = arr.shape[1] * 8
    return [int.from_bytes(b[i:i + w], "little") for i in range(0, len(b), w)]


def ntt_inputs(curve, log_n, seed):
    """Uniform Montgomery limbs in [0, p) with planted runs of the limb values p - 1, 0, 1 and of the elements -1 and 1."""
    f = curve.fr
    n = 1 << log_n
    x = uniform_below(np.random.default_rng(seed), n, f.p)
    run = max(1, n >> 6)
    planted = [f.p - 1, 0, 1, f.to_mont(f.p - 1), f.to_mont(1)]
    for k, v in enumerate(planted):
        at = (2 * k + 1) * n // (2 * len(planted) + 1)
        x[at:at + run] = _modulus_limbs(v, 4)
    x[-1] = _modulus_limbs(f.p - 1, 4)
    return x


def gpu_ntt(ctx, curve, data, log_n, inverse, coset):
    out = np.ascontiguousarray(data.copy())
    _lib.check(_lib.lib().b2m_ntt(ctx, util.CURVE_ID[curve.name], _lib.ptr(out), log_n, inverse, coset))
    assert below(out, curve.fr.p).all(), ("output not fully reduced", curve.name, log_n, inverse, coset)
    return out


def check_four_modes(ctx, curve, x, log_n):
    """fft and coset fft equal cport's; the inverse transforms of cport's outputs give back x, limb for limb."""
    for coset, ref in ((0, cport.fft), (1, cport.coset_fft)):
        want = ref(curve.name, x.copy())
        assert np.array_equal(gpu_ntt(ctx, curve, x, log_n, 0, coset), want), (curve.name, log_n, "forward", coset)
        assert np.array_equal(gpu_ntt(ctx, curve, want, log_n, 1, coset), x), (curve.name, log_n, "inverse", coset)
        del want


def new_ctx():
    h = ctypes.c_void_p()
    _lib.check(_lib.lib().b2m_ctx_create(0, ctypes.byref(h)))
    return h


@pytest.fixture(scope="module")
def nctx():
    """A context of this module's own, so that the 2^27 twiddle table it grows goes away with it."""
    h = new_ctx()
    yield h
    _lib.lib().b2m_ctx_destroy(h)


# ---- NTT ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("curve", CURVES, ids=lambda c: c.name)
@pytest.mark.parametrize("log_n", [17, 19, 23, 24, 25])
def test_ntt_three_and_four_passes_match_cport(nctx, curve, log_n):
    """Three passes (9+8 at 2^17, 7+6+6 at 2^19, 8+8+7 at 2^23, 8+8+8 at 2^24) and four (7+6+6+6 at 2^25)."""
    check_four_modes(nctx, curve, ntt_inputs(curve, log_n, 1000 + log_n), log_n)


@pytest.mark.parametrize("curve,log_n", [(BLS12_381, 26), (BN254, 26), (BLS12_381, 27)], ids=["bls12_381-26", "bn254-26", "bls12_381-27"])
def test_ntt_prover_sizes_match_cport(nctx, curve, log_n):
    """The 2^24-constraint prover's largest transforms (|K| = 2^26, and 2^27 for its quotient)."""
    nbytes = 32 << log_n
    _require_memory(3 * nbytes + (nbytes >> 1) + (4 << 30), 4 * nbytes + (4 << 30))
    check_four_modes(nctx, curve, ntt_inputs(curve, log_n, 2000 + log_n), log_n)


@pytest.mark.parametrize("curve", CURVES, ids=lambda c: c.name)
@pytest.mark.parametrize("log_n", [17, 23])
def test_ntt_delta_at_last_index(nctx, curve, log_n):
    """A single non-zero coefficient, at n - 1: every output is a distinct power of the root (or of g times it)."""
    f = curve.fr
    x = np.zeros((1 << log_n, 4), dtype=np.uint64)
    x[-1] = _modulus_limbs(f.to_mont(f.p - 2), 4)
    check_four_modes(nctx, curve, x, log_n)


def test_ntt_small_transforms_read_a_strided_twiddle_table():
    """On a fresh context, one 2^25 transform grows the twiddle table first; every transform of 2^0 to 2^16 after it reads
    that table at a stride of 2^(25 - log_n) (sh > 0), and must still equal the Python Domain in all four modes."""
    ctx = new_ctx()
    try:
        for curve in CURVES:
            gpu_ntt(ctx, curve, ntt_inputs(curve, 25, 7), 25, 0, 0)
        for curve in CURVES:
            f = curve.fr
            for log_n in range(17):
                n = 1 << log_n
                vals = limbs_to_ints(uniform_below(np.random.default_rng(300 + log_n), n, f.p))
                vals[-1] = 1
                vals[0] = f.p - 1
                d = Domain(f, n)
                xm = util.fr_to_mont_limbs(curve, vals)
                for inverse, coset in ((0, 0), (1, 0), (0, 1), (1, 1)):
                    want = {(0, 0): d.fft, (1, 0): d.ifft, (0, 1): d.coset_fft, (1, 1): d.coset_ifft}[(inverse, coset)](vals)
                    got = gpu_ntt(ctx, curve, xm, log_n, inverse, coset)
                    assert np.array_equal(got, util.fr_to_mont_limbs(curve, want)), (curve.name, log_n, inverse, coset)
    finally:
        _lib.lib().b2m_ctx_destroy(ctx)


@pytest.mark.parametrize("curve,log_n", [(BN254, 29), (BLS12_381, 33)], ids=["bn254-29", "bls12_381-33"])
def test_ntt_above_two_adicity_is_rejected_without_allocating(nctx, curve, log_n):
    L = _lib.lib()
    mem = (ctypes.c_size_t * 3)()
    _lib.check(L.b2m_ctx_memory(nctx, mem))
    in_use = mem[0]
    buf = np.zeros((4, 4), dtype=np.uint64)
    for inverse, coset in ((0, 0), (1, 1)):
        with pytest.raises(_lib.B2MError) as ei:
            _lib.check(L.b2m_ntt(nctx, util.CURVE_ID[curve.name], _lib.ptr(buf), log_n, inverse, coset))
        assert ei.value.code == ERR_DEGREE_TOO_LARGE
    _lib.check(L.b2m_ctx_memory(nctx, mem))
    assert mem[0] == in_use and mem[1] == in_use, "a rejected transform allocated device memory"
    assert not buf.any()


# ---- MSM ---------------------------------------------------------------------------------------------------------------------

def srs_msm(srs, curve, off, sc_limbs):
    """b2m_srs_msm over canonical scalar limbs -> affine point or None; the output coordinates must be fully reduced."""
    out = np.zeros(2 * curve.fq.limbs64, dtype=np.uint64)
    inf = ctypes.c_int(0)
    sc = np.ascontiguousarray(sc_limbs, dtype=np.uint64)
    _lib.check(_lib.lib().b2m_srs_msm(srs, off, _lib.ptr(sc), len(sc), _lib.ptr(out), ctypes.byref(inf)))
    assert below(out, curve.fq.p).all()
    P = util.points_from_limbs(curve, out)[0]
    assert (P is None) == bool(inf.value)
    return P


def trapdoor(curve, beta, off, sc_limbs):
    """(sum_i s_i beta^(off + i)) g, by Horner over the scalars."""
    r = curve.fr.p
    acc = 0
    for s in reversed(limbs_to_ints(sc_limbs)):
        acc = (acc * beta + s) % r
    return ec.scalar_mul(curve, acc * pow(beta, off, r) % r, curve.g)


def check_msm(ctx, curve, n, scalar_sets, window_bits=0, beta=0x2f8a9b1c3d4e5f60718293a4b5c6d7e8f9):
    """A fresh SRS of n powers beta^i g; each (offset, scalars) equals the trapdoor's answer."""
    beta %= curve.fr.p
    srs = util.make_srs(ctx, curve, util.gpu_powers(ctx, curve, curve.g, beta, n), window_bits=window_bits)
    try:
        for off, sc in scalar_sets:
            assert srs_msm(srs, curve, off, sc) == trapdoor(curve, beta, off, sc), (curve.name, n, window_bits, off)
    finally:
        _lib.lib().b2m_srs_destroy(srs)


@pytest.mark.parametrize("log_n", [21, 23])
def test_msm_bn254_xyzz_only_at_scale(b2m_ctx, log_n):
    """BN254's default bucket pass has no batched-affine levels: the accumulate and stitch kernels see all W n references
    (c = 20 at these sizes)."""
    n = 1 << log_n
    sc = uniform_below(np.random.default_rng(log_n), n, BN254.fr.p)
    check_msm(b2m_ctx, BN254, n, [(0, sc)])


def test_msm_bls12_381_levels_off_at_scale(b2m_ctx, monkeypatch):
    monkeypatch.setenv("B2M_MSM_AFFINE_LEVELS", "0")
    n = 1 << 23
    sc = uniform_below(np.random.default_rng(23), n, BLS12_381.fr.p)
    check_msm(b2m_ctx, BLS12_381, n, [(0, sc)])


@pytest.mark.parametrize("curve", CURVES, ids=lambda c: c.name)
def test_msm_short_stitch_queue_overflows(b2m_ctx, monkeypatch, curve):
    """More runs of 3+ accumulate threads than the short queue holds: the runs past its capacity are folded serially by the
    stitch thread that found them.  c = 20, n = 2^22: each of the 12 full windows (bits 0-239) takes its digit from one pool
    of P distinct positive digits <= 2^19 (no sign carries, top window 0, so every scalar is < 2^240 < r), every digit used
    equally often; each used bucket then holds more than 2 q references and spans at least three threads."""
    monkeypatch.setenv("B2M_MSM_AFFINE_LEVELS", "0")
    c, W_full, n = 20, 12, 1 << 22
    P = 280_000
    refs_per_bucket = W_full * n // P
    assert P > LONG_CAP and refs_per_bucket > 2 * Q_BOUND, "the case no longer overflows the short stitch queue"
    rng = np.random.default_rng(int(curve.name == "bn254"))
    pool = rng.choice(np.arange(1, (1 << (c - 1)) + 1, dtype=np.uint64), size=P, replace=False)
    digits = rng.permutation(np.resize(pool, W_full * n)).reshape(n, W_full)
    sc = np.zeros((n, 4), dtype=np.uint64)
    for w in range(W_full):
        bit = c * w
        limb, off = bit // 64, bit % 64
        d = digits[:, w]
        sc[:, limb] |= d << np.uint64(off)
        if off + c > 64:
            sc[:, limb + 1] |= d >> np.uint64(64 - off)
    del digits
    check_msm(b2m_ctx, curve, n, [(0, sc)], window_bits=c)


@pytest.mark.parametrize("curve", CURVES, ids=lambda c: c.name)
@pytest.mark.parametrize("c", [17, 18, 19, 21, 22, 23, 24])
def test_msm_wide_windows(b2m_ctx, curve, c):
    """Window widths the picker never chooses: 24 has 2^23 buckets and the widest reduction (L = 4096, R = 2048); 21 and 23
    leave a top window of 4 and 3 bits that sends all n references into a handful of buckets."""
    n = 1 << 18
    r = curve.fr.p
    rng = np.random.default_rng(c)
    uni = uniform_below(rng, n, r)
    same = np.tile(uniform_below(rng, 1, r), (n, 1))
    alt = np.tile(_modulus_limbs(r - 1, 4), (n, 1))
    alt[1::2] = _modulus_limbs(r - 2, 4)
    check_msm(b2m_ctx, curve, n, [(0, uni), (0, same), (0, alt), (77, uni[:n // 2 + 1])], window_bits=c)


def test_msm_bn254_2p24(b2m_ctx):
    """2^24 uniform scalars: ~384 references per bucket at c = 20, so more than 2^19 runs of 10-14 slots split between the
    two stitch queues."""
    n = 1 << 24
    _require_memory(20 * 10 ** 9, 8 << 30)
    sc = uniform_below(np.random.default_rng(24), n, BN254.fr.p)
    check_msm(b2m_ctx, BN254, n, [(0, sc)])


@pytest.mark.parametrize("curve", CURVES, ids=lambda c: c.name)
@pytest.mark.parametrize("log_n", [16, 18])
def test_msm_g1_one_shot_matches_cport(b2m_ctx, curve, log_n):
    """`b2m_msm_g1` on arbitrary host bases (i + 1) g, with the point at infinity, repeated points and a point next to its
    negation planted among them, equals cport's Pippenger limb for limb."""
    fq = curve.fq
    lq = fq.limbs64
    n = 1 << log_n
    g = util.points_to_limbs(curve, [curve.g])
    bases = np.zeros((n, 2 * lq), dtype=np.uint64)
    cport.lib().cport_gen_bases(cport.CURVE_ID[curve.name], cport._ptr(g), n, cport._ptr(bases))
    bases[5] = 0                          # infinity
    bases[n // 2] = 0
    bases[100:164] = bases[99]            # repeated points
    bases[n - 40:n - 8] = bases[7]
    y = limbs_to_ints(bases[1000:1001, lq:])[0]
    bases[1001, :lq] = bases[1000, :lq]   # -P right after P
    bases[1001, lq:] = _modulus_limbs(fq.p - y, lq)
    sc = uniform_below(np.random.default_rng(log_n), n, curve.fr.p)
    sc[1000] = sc[1001]                   # so that P and -P cancel in every window
    sc[200:260] = 0
    want = cport.msm(curve.name, bases, sc)
    out = np.zeros(2 * lq, dtype=np.uint64)
    inf = ctypes.c_int(0)
    _lib.check(_lib.lib().b2m_msm_g1(b2m_ctx, util.CURVE_ID[curve.name], _lib.ptr(bases), _lib.ptr(sc), n, _lib.ptr(out), ctypes.byref(inf)))
    assert below(out, fq.p).all() and not inf.value
    assert np.array_equal(out, want)
