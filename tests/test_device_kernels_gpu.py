"""GPU: single device kernels compared one to one with Python integers, at the inputs that reach their edge cases.

Whole proofs and the Level-0 ABI check the CUDA code only in aggregate; here each kernel runs alone through
tests/gpu/libb2m_kernel_tests.so (the product's headers behind a test-only C ABI, built by __graft_entry__.build())
or through the Level-0 ABI with chosen scalars, and every expected value comes from Python integers or the oracle:

  A  field arithmetic (PTX carry chains, `__ffs` in inverse_fast) on all four fields
  B  the XYZZ group law and to_affine on device threads
  C  exclusive_scan_u32 around block and recursion boundaries
  D  rec_suffix (division by X - z, Horner, division by X^s - 1, segmented sums) at recursion depths 1-3
  E  batch_inverse (zeros skipped) and spmv_kernel (empty rows, repeated columns, long rows)
  F  the mask sampler's attempt kernel at every stream offset mod 16 and across block counter 2^32
  G  whole proofs whose zk stream starts off the 8-word grid, ChaCha8/12/20, against oracle/cport's prover
  H  MSM signed-digit recoding at every window width 8..24, and at the benchmark's c = 20 with default knobs
"""
import ctypes
import os
import random

import numpy as np
import pytest

from oracle import ec
from oracle import rng as orng
from oracle.params import BLS12_381, BN254, BLS12_381_FR, BLS12_381_FQ, BN254_FR, BN254_FQ

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
SHIM = os.path.join(HERE, "gpu", "libb2m_kernel_tests.so")
CURVES = [BLS12_381, BN254]
FIELDS = [BLS12_381_FR, BLS12_381_FQ, BN254_FR, BN254_FQ]  # kernel_shim.cu field ids 0..3
OP_MUL, OP_ADD, OP_SUB, OP_NEG, OP_INV, OP_TO_CANON, OP_FROM_CANON, OP_INV_FAST, OP_SQR, OP_DBL, OP_POW_U64 = range(11)


@pytest.fixture(scope="module")
def kt():
    if not os.path.exists(SHIM):
        pytest.fail(f"{SHIM} is missing: run __graft_entry__.build(), which builds it with `make -C tests/gpu`")
    L = ctypes.CDLL(SHIM)
    vp, sz, ci, u64 = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_uint64
    L.kt_last_error.restype = ctypes.c_char_p
    L.kt_ctx_create.argtypes = [ci]
    L.kt_ctx_destroy.restype = None
    L.kt_field_op.argtypes = [ci, ci, vp, vp, sz, vp]
    L.kt_curve_op.argtypes = [ci, ci, vp, vp, ci, sz, vp, ci, vp]
    L.kt_scan_u32.argtypes = [vp, sz, vp]
    L.kt_rec_suffix.argtypes = [ci, vp, sz, sz, vp, ci, ci, vp]
    L.kt_batch_inverse.argtypes = [ci, vp, sz]
    L.kt_spmv.argtypes = [ci, vp, vp, vp, vp, sz, vp]
    L.kt_sample.argtypes = [ci, vp, ci, u64, sz, vp, vp]
    _check(L, L.kt_ctx_create(0))
    yield L
    L.kt_ctx_destroy()


def _check(L, rc):
    if rc != 0:
        raise RuntimeError(f"kernel test library error {rc}: {L.kt_last_error().decode()}")


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def n32_of(field):
    return 8 if field.bits <= 256 else 12


def to_u32(vals, n32):
    """python ints -> (len, n32) little-endian uint32 limbs"""
    buf = b"".join(int(v).to_bytes(4 * n32, "little") for v in vals)
    return np.frombuffer(buf, dtype=np.uint32).reshape(len(vals), n32).copy()


def from_u32(arr):
    arr = np.ascontiguousarray(arr, dtype=np.uint32)
    w = 4 * arr.shape[-1]
    raw = arr.tobytes()
    return [int.from_bytes(raw[i:i + w], "little") for i in range(0, len(raw), w)]


def rand_below_half(rnd_np, n, field):
    """n random elements < 2^(bits - 1) < p as uint32 limbs (cheap to draw in bulk; valid Montgomery representatives)"""
    n32 = n32_of(field)
    a = rnd_np.integers(0, 1 << 32, size=(n, n32), dtype=np.uint64).astype(np.uint32)
    top = field.bits - 1 - 32 * (n32 - 1)
    a[:, n32 - 1] &= np.uint32((1 << top) - 1)
    return a


# ---------------------------------------------------------------------------------------------------
# A. field arithmetic on the device
# ---------------------------------------------------------------------------------------------------
def edge_values(p, n32):
    R = 1 << (32 * n32)
    bits = p.bit_length()
    vals = [0, 1, 2, 3, p - 1, p - 2, p - 3, R % p, R * R % p, pow(R, -1, p), p - R % p, (p - 1) // 2, (p + 1) // 2, (p + 3) // 2,
            0xffffffff, (1 << 64) - 1, (1 << 64) + (1 << 33), (1 << (bits - 1)) - 1]
    vals += [1 << k for k in (1, 31, 32, 33, 63, 64, 65, 127, 128, 191, 192, bits - 2, bits - 1) if (1 << k) < p]
    vals += [p - (1 << k) for k in (0, 1, 31, 32, 64, 128, bits - 2) if (1 << k) < p]
    out = []
    for v in vals:
        if 0 <= v < p and v not in out:
            out.append(v)
    return out


def carry_pairs(p, n32, rnd, count):
    """Operands whose partial products have a low word of 0xffffffff: a's top limb t is odd and b's other limbs are
    -t^-1 mod 2^32, so each row's last `madc.lo.cc` of the shifted accumulation can carry into its closing `madc.hi`
    (random operands almost never do: that carry-in is then 0, and a carry chain that dropped it would go unseen)."""
    top = p >> (32 * (n32 - 1))
    out = []
    for _ in range(count):
        t = rnd.randrange(1, top) | 1
        w = (-pow(t, -1, 1 << 32)) % (1 << 32)
        a = (t << (32 * (n32 - 1))) | rnd.getrandbits(32 * (n32 - 1))
        b = sum(w << (32 * i) for i in range(n32 - 1)) | (rnd.randrange(top) << (32 * (n32 - 1)))
        out += [(a, b), (b, a)]
    return out


@pytest.mark.parametrize("fi", range(4), ids=[f.name for f in FIELDS])
def test_field_ops_device(kt, fi):
    """Every op of field.cuh on device threads, element for element against Python integers: all pairs of edge values,
    operands whose results are 0, 1 and p-1, operands that drive carries into the closing `madc.hi` of a multiplier
    row, and 2^16 random pairs.  The multiplication is also checked against the
    unreduced CIOS value t = (ab + mp) / R, and the inputs are asserted to reach both sides of its final subtraction."""
    field = FIELDS[fi]
    p = field.p
    n32 = n32_of(field)
    R = 1 << (32 * n32)
    Rinv = pow(R, -1, p)
    rnd = random.Random(1000 + fi)
    E = edge_values(p, n32)
    A = [a for a in E for _ in E]
    B = [b for _ in E for b in E]
    for target in (0, 1, p - 1):
        for _ in range(64):
            a = rnd.randrange(1, p)
            A += [a, a, a]
            B += [target * R * pow(a, -1, p) % p, (target - a) % p, (a - target) % p]  # a*b/R, a+b, a-b == target
    for a, b in carry_pairs(p, n32, rnd, 2048):
        A.append(a)
        B.append(b)
    for _ in range(1 << 16):
        A.append(rnd.randrange(p))
        B.append(rnd.randrange(p))
    n = len(A)
    a_l, b_l = to_u32(A, n32), to_u32(B, n32)
    out = np.zeros_like(a_l)

    def run(op, b=b_l):
        _check(kt, kt.kt_field_op(fi, op, _p(a_l), _p(b), n, _p(out)))
        return from_u32(out)

    got = run(OP_MUL)
    pinv_neg = (-pow(p, -1, R)) % R
    hi = lo = 0
    for a, b, g in zip(A, B, got):
        t = (a * b + (a * b * pinv_neg % R) * p) >> (32 * n32)
        assert g == (t - p if t >= p else t) == a * b * Rinv % p, (hex(a), hex(b))
        hi += t >= p
        lo += t < p
    assert hi and lo, (hi, lo)
    assert run(OP_SQR) == [a * a * Rinv % p for a in A]
    assert run(OP_ADD) == [(a + b) % p for a, b in zip(A, B)]
    assert run(OP_SUB) == [(a - b) % p for a, b in zip(A, B)]
    assert run(OP_NEG) == [(-a) % p for a in A]
    assert run(OP_DBL) == [2 * a % p for a in A]
    assert run(OP_TO_CANON) == [a * Rinv % p for a in A]
    assert run(OP_FROM_CANON) == [a * R % p for a in A]
    # a Montgomery inverse is a^-1 * R^2 as an integer; inverse(0) = 0 for both ladders
    inv = [pow(a, -1, p) * R * R % p if a else 0 for a in A]
    assert run(OP_INV) == inv
    assert run(OP_INV_FAST) == inv
    # pow_u64: exponent = the low 64 bits of b (0 and 1 included); in Montgomery form x^e = (a/R)^e * R
    exps = [0, 1, 2, 3, (1 << 64) - 1, 1 << 63, p - 2 & ((1 << 64) - 1)] + [rnd.getrandbits(64) for _ in range(n - 7)]
    e_l = to_u32(exps, n32)
    assert run(OP_POW_U64, e_l) == [pow(a * Rinv % p, e, p) * R % p for a, e in zip(A, exps)]

    # inverse_fast on the host test's special values: powers of two and long runs of trailing zeros (the ctz/__ffs path)
    bits = p.bit_length()
    special = [1, 2, 3, 4, p - 1, p - 2, (p - 1) // 2, (p + 1) // 2, R % p, R * R % p, 1 << 32, 1 << 64, (1 << 64) + (1 << 33),
               1 << (bits - 1), (1 << (bits - 1)) - 1, p - (1 << 40), 0xffffffff, 0xffffffff00000000, 0]
    special += [(1 << k) % p for k in range(1, 32 * n32)] + [p - ((1 << k) % p) for k in range(1, 32 * n32, 7)]
    special += [(rnd.randrange(1, 1 << 40) << k) % p for k in range(32, bits - 41, 5)]
    a_l = to_u32(special, n32)
    out = np.zeros_like(a_l)
    _check(kt, kt.kt_field_op(fi, OP_INV_FAST, _p(a_l), _p(a_l), len(special), _p(out)))
    assert from_u32(out) == [pow(a, -1, p) * R * R % p if a else 0 for a in special]


# ---------------------------------------------------------------------------------------------------
# B. XYZZ on the device
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ci,curve", list(enumerate(CURVES)), ids=[c.name for c in CURVES])
def test_xyzz_device(kt, ci, curve):
    """add_mixed, full add (doubling and cancellation reached through `add`), scalar_mul and to_affine on device threads,
    with P + P, P - P, O + P and P + O, against oracle/ec.py in affine form."""
    fq, r = curve.fq, curve.fr.p
    n32 = n32_of(fq)
    rnd = random.Random(50 + ci)

    def pack(pt_lists):
        vals = []
        for pts in pt_lists:
            for P in pts:
                vals += [0, 0] if P is None else [fq.to_mont(P[0]), fq.to_mont(P[1])]
        return to_u32(vals, n32)

    def unpack(arr):
        v = from_u32(np.asarray(arr).reshape(-1, n32))  # x, y, x, y, ...
        return [None if v[2 * i] == 0 and v[2 * i + 1] == 0 else (fq.from_mont(v[2 * i]), fq.from_mont(v[2 * i + 1])) for i in range(len(v) // 2)]

    def run(which, cases, negs, ks=None):
        npts = len(cases[0])
        pts = pack(cases)
        ng = np.array(negs, dtype=np.uint8).reshape(-1)
        k = None if ks is None else to_u32(ks, 8)
        out = np.zeros((len(cases), 2 * n32), dtype=np.uint32)
        _check(kt, kt.kt_curve_op(ci, which, _p(pts), _p(ng), npts, len(cases), _p(k), 8, _p(out)))
        return unpack(out)

    def expect(pts, neg):
        acc = None
        for P, s in zip(pts, neg):
            acc = ec.affine_add(curve, acc, ec.affine_neg(curve, P) if s else P)
        return acc

    base = [ec.scalar_mul(curve, rnd.randrange(1, r), curve.g) for _ in range(12)]
    P, Q = base[0], base[1]
    nP = ec.affine_neg(curve, P)
    # two-point cases: with `which` = 1 the pair meets in one full addition (point 0 -> b, point 1 -> a, then a.add(b))
    pairs = [([P, P], [0, 0]), ([P, P], [0, 1]), ([P, P], [1, 1]), ([P, nP], [0, 0]), ([nP, P], [1, 0]), ([None, P], [0, 0]),
             ([P, None], [0, 0]), ([None, None], [0, 0]), ([None, P], [1, 1]), ([P, Q], [0, 1]), ([Q, P], [0, 0])]
    cases = [c for c, _ in pairs]
    negs = [n for _, n in pairs]
    want = [expect(c, n) for c, n in pairs]
    assert want[1] is None and want[3] is None and want[7] is None and want[0] == ec.scalar_mul(curve, 2, P)
    for which in (0, 1):
        assert run(which, cases, negs) == want, which
    # longer sums with doublings, cancellations and infinity inside them
    long_cases, long_negs = [], []
    for _ in range(32):
        pts = base[2:12] + [base[2], base[3], ec.affine_neg(curve, base[4]), None, base[2]]
        rnd.shuffle(pts)
        long_cases.append(pts)
        long_negs.append([rnd.randrange(2) for _ in pts])
    want = [expect(c, n) for c, n in zip(long_cases, long_negs)]
    for which in (0, 1):
        assert run(which, long_cases, long_negs) == want, which
    # scalar_mul (double-and-add through dbl and add_mixed), including 0, 1, r-1 and the point at infinity
    ks = [0, 1, 2, 3, r - 1, r - 2, (r + 1) // 2, 1 << 128] + [rnd.randrange(r) for _ in range(8)] + [5, 0]
    pts = [[P]] * (len(ks) - 2) + [[None], [None]]
    got = run(2, pts, [[0]] * len(pts), ks)
    assert got == [None if pt[0] is None else ec.scalar_mul(curve, k, pt[0]) for pt, k in zip(pts, ks)]


# ---------------------------------------------------------------------------------------------------
# C. exclusive_scan_u32
# ---------------------------------------------------------------------------------------------------
SCAN_SIZES = [0, 1, 2, 2047, 2048, 2049, 2048 * 2048 - 1, 2048 * 2048, 2048 * 2048 + 1] + [(1 << (c - 1)) + 1 for c in (8, 16, 20, 24)]


@pytest.mark.parametrize("n", SCAN_SIZES)
def test_exclusive_scan(kt, n):
    """One block is 512 threads x 4 items = 2048; 2048^2 + 1 is where the recursion gains its second level, and the
    B + 1 = 2^(c-1) + 1 bucket counts of the MSM reach three levels at c = 24.  Totals that wrap mod 2^32 included."""
    rng = np.random.default_rng(n)
    inputs = {"zeros": np.zeros(n, dtype=np.uint32), "ones": np.ones(n, dtype=np.uint32),
              "random": rng.integers(0, 1 << 12, size=n, dtype=np.uint64).astype(np.uint32),
              "wrapping": rng.integers((1 << 32) - (1 << 20), 1 << 32, size=n, dtype=np.uint64).astype(np.uint32)}
    for name, x in inputs.items():
        out = np.full(n, 0xdeadbeef, dtype=np.uint32)
        _check(kt, kt.kt_scan_u32(_p(x), n, _p(out)))
        want = np.zeros(n, dtype=np.uint64)  # (all-uint64: a mixed int64 / uint64 concatenation would round through float64)
        want[1:] = np.cumsum(x.astype(np.uint64))[:-1]
        want &= np.uint64(0xffffffff)
        assert np.array_equal(out.astype(np.uint64), want), name


# ---------------------------------------------------------------------------------------------------
# D. rec_suffix
# ---------------------------------------------------------------------------------------------------
REC_SIZES = [1, 31, 32, 33, 1023, 1024, 1025, 32769, (1 << 20) + 3]


def rec_reference(vals, s, zz, mul, p):
    """out[j] = in[j] + z * out[j + s] (plain sum when not mul), out[j >= n] = 0, in the Montgomery domain:
    zz = z_mont / R, so zz * out_mont is the Montgomery product."""
    n = len(vals)
    out = list(vals)
    for j in range(n - s - 1, -1, -1):
        out[j] = (out[j] + (zz * out[j + s] if mul else out[j + s])) % p
    return out


@pytest.mark.parametrize("ci,curve", list(enumerate(CURVES)), ids=[c.name for c in CURVES])
@pytest.mark.parametrize("n", REC_SIZES)
def test_rec_suffix(kt, ci, curve, n):
    """n / s just above REC_M = 32, 32^2 and 32^3 super-elements (recursion depth 1-3), s larger than n, z in {0, 1, p-1,
    random}, the `mul = false` form, in place and out of place.  The 2^20 + 3 case is checked in full."""
    f = curve.fr
    p = f.p
    R = 1 << 256
    Rinv = pow(R, -1, p)
    rnd = random.Random(n * 7 + ci)
    vals_l = rand_below_half(np.random.default_rng(n + ci), n, f)
    vals_l[0] = to_u32([p - 1], 8)[0]
    vals_l[-1] = to_u32([p - 1], 8)[0]
    if n > 2:
        vals_l[n // 2] = 0
    vals = from_u32(vals_l)
    big = n > 40000
    strides = [1, 2, 3, 32, 33, 64, 1024, n - 1, n, n + 1]
    if big:
        strides = [1, 3, 33, 1024, n + 1]
    strides = sorted({s for s in strides if s >= 1})
    zs = [0, 1, p - 1, rnd.randrange(p)]
    cases = []
    for s in strides:
        if big:
            cases += [(s, rnd.randrange(p), True), (s, p - 1, True)] if s in (1, 33) else [(s, rnd.randrange(p), True)]
        else:
            cases += [(s, z, True) for z in zs]
        cases.append((s, 0, False))
    if big:
        cases += [(1, 0, True), (1, 1, True)]
    for k, (s, z, mul) in enumerate(cases):
        zm = f.to_mont(z)
        want = rec_reference(vals, s, zm * Rinv % p, mul, p)
        for in_place in ((k % 2 == 0,) if big else (False, True)):
            out = np.zeros_like(vals_l)
            _check(kt, kt.kt_rec_suffix(ci, _p(vals_l), n, s, _p(to_u32([zm], 8)), int(mul), int(in_place), _p(out)))
            got = from_u32(out)
            if got != want:
                bad = next(j for j in range(n) if got[j] != want[j])
                pytest.fail(f"n={n} s={s} z={z} mul={mul} in_place={in_place}: first mismatch at {bad}")


# ---------------------------------------------------------------------------------------------------
# E. batch_inverse and spmv
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ci,curve", list(enumerate(CURVES)), ids=[c.name for c in CURVES])
def test_batch_inverse(kt, ci, curve):
    """Montgomery's trick over BINV_M = 32 strided elements per thread: lengths around 32 and 4096 threads, zeros first,
    last, at every 32nd position and everywhere; zeros come back as zeros, everything else as its inverse."""
    f = curve.fr
    p = f.p
    R = 1 << 256
    rnd = random.Random(70 + ci)
    for n in (1, 2, 31, 32, 33, 4095, 32 * 4096 + 1):
        base = [rnd.randrange(1, p) for _ in range(n)]
        base[0] = 1 % p
        if n > 1:
            base[1] = p - 1
        if n > 2:
            base[2] = R % p  # Montgomery one
        layouts = {"none": base, "first": [0] + base[1:], "last": base[:-1] + [0], "every_32nd": [0 if j % 32 == 0 else v for j, v in enumerate(base)],
                   "every_33rd": [0 if j % 33 == 5 else v for j, v in enumerate(base)], "all": [0] * n}
        for name, vals in layouts.items():
            data = to_u32(vals, 8)
            _check(kt, kt.kt_batch_inverse(ci, _p(data), n))
            assert from_u32(data) == [pow(v, -1, p) * R * R % p if v else 0 for v in vals], (n, name)


@pytest.mark.parametrize("ci,curve", list(enumerate(CURVES)), ids=[c.name for c in CURVES])
def test_spmv(kt, ci, curve):
    """CSR z_A = A z as the prover launches it: empty rows (leading, inner, trailing), repeated columns inside a row, one
    row of 10^4 entries, coefficients 0 and p-1."""
    f = curve.fr
    p = f.p
    R = 1 << 256
    Rinv = pow(R, -1, p)
    rnd = random.Random(90 + ci)
    nz = 3000
    z = [rnd.randrange(p) for _ in range(nz)]
    z[0], z[1], z[2] = 0, p - 1, R % p
    rows = [[], [], [(5, p - 1)], [(7, 0), (7, 1), (7, p - 1)], [], [(nz - 1, rnd.randrange(p))] * 4]
    rows.append([(rnd.randrange(nz), rnd.choice([0, p - 1, R % p, rnd.randrange(p)])) for _ in range(10 ** 4)])
    rows += [[(rnd.randrange(nz), rnd.randrange(p)) for _ in range(rnd.randrange(0, 6))] for _ in range(700)]
    rows += [[(1, p - 1), (1, p - 1), (0, 3)], [], [], []]
    row_ptr = [0]
    col, coeff = [], []
    for row in rows:
        for c, v in row:
            col.append(c)
            coeff.append(v)
        row_ptr.append(len(col))
    out = np.zeros((len(rows), 8), dtype=np.uint32)
    _check(kt, kt.kt_spmv(ci, _p(np.array(row_ptr, dtype=np.uint32)), _p(np.array(col, dtype=np.uint32)), _p(to_u32(coeff, 8)),
                          _p(to_u32(z, 8)), len(rows), _p(out)))
    want = [sum(v * z[c] for c, v in row) * Rinv % p for row in rows]  # Montgomery products summed
    assert from_u32(out) == want


# ---------------------------------------------------------------------------------------------------
# F. mask sampler, kernel level
# ---------------------------------------------------------------------------------------------------
SAMPLE_POS = list(range(16)) + [16 * 1000 + 9, (1 << 36) - 40, (1 << 36) - 43]


@pytest.mark.parametrize("ci,curve", list(enumerate(CURVES)), ids=[c.name for c in CURVES])
@pytest.mark.parametrize("rounds", [8, 12, 20])
def test_sample_attempts(kt, ci, curve, rounds):
    """sample_attempts_kernel: attempt a is the `F::rand` draw at word pos0 + 8a.  pos0 = 9..15 (mod 16) makes every other
    attempt straddle two ChaCha blocks (the second-block path); 2^36 - 40 and 2^36 - 43 cross block counter 2^32 (state
    word 13), the latter inside a straddling attempt."""
    f = curve.fr
    seed = bytes((7 * i + 3 * ci + rounds) & 0xff for i in range(32))
    key = np.frombuffer(seed, dtype=np.uint8).copy()
    na = 40
    top_mask = (1 << (64 - f.repr_shave_bits)) - 1
    for pos0 in SAMPLE_POS:
        cand = np.zeros((na, 8), dtype=np.uint32)
        acc = np.zeros(na, dtype=np.uint32)
        _check(kt, kt.kt_sample(ci, _p(key), rounds, pos0, na, _p(cand), _p(acc)))
        got = from_u32(cand)
        for a in range(na):
            g = orng.ChaChaRng(seed, rounds, word_pos=pos0 + 8 * a)
            limbs = [g.next_u64() for _ in range(4)]
            limbs[-1] &= top_mask
            v = sum(l << (64 * i) for i, l in enumerate(limbs))
            assert (got[a], int(acc[a])) == (v, int(v < f.p)), (pos0, a)


# ---------------------------------------------------------------------------------------------------
# G. mask sampler, whole proof
# ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gctx(b2m_ctx):
    from marlin_b200 import api
    c = api.Context.__new__(api.Context)
    c.handle = b2m_ctx
    return c


@pytest.mark.parametrize("curve_name,scheme,log_n,rounds,pos0", [
    ("bls12_381", "marlin_kzg10", 8, 8, 1),
    ("bls12_381", "sonic_kzg10", 9, 20, 9),
    ("bls12_381", "marlin_kzg10", 10, 12, 15),
    ("bls12_381", "sonic_kzg10", 8, 8, 12),
    ("bls12_381", "marlin_kzg10", 9, 20, (1 << 36) - 40),
    ("bn254", "marlin_kzg10", 13, 20, 4),  # 3|H| draws at acceptance ~0.76 need a second sampler pass
    ("bn254", "marlin_kzg10", 8, 12, (1 << 36) - 43),
])
def test_prove_zk_stream_offsets(gctx, curve_name, scheme, log_n, rounds, pos0):
    """A caller's zk rng is rarely at word 0: the reference's own test draws SRS and circuit values from it first.  From a
    start off the 8-word grid the mask polynomial's attempts straddle ChaCha blocks; proof bytes and the final stream
    position must equal oracle/cport's C++ prover from the same (seed, rounds, word_pos)."""
    from marlin_b200 import api, r1cs as gr1cs
    from oracle import cport
    n = 1 << log_n
    cid = 0 if curve_name == "bls12_381" else 1
    a, b = 0x1234567890abcdef1234567890abcdef, 0xfedcba0987654321fedcba0987654321
    m = api.Marlin(curve_name, scheme, ctx=gctx)
    srs = m.universal_setup(n, n, 3 * n, beta=0x5eed5eed5eed5eed5eed5eed, gamma=7, degree_bounds=(n - 2, 4 * n - 2))
    circ = gr1cs.dummy_circuit(cid, a, b, 10, n)
    seed = bytes((31 * i + rounds) & 0xff for i in range(32))
    try:
        pk = m.index(srs, circ)
        try:
            rng = api.ZkRng(seed, rounds, word_pos=pos0)
            gproof = m.prove(pk, circ, rng)
            cp = cport.CpuProver(curve_name, scheme, srs.powers_limbs, srs.gamma_limbs, srs.gamma_indices, circ.num_constraints,
                                 circ.num_variables, circ.num_instance, circ.a, circ.b, circ.c)
            try:
                assert cp.vk_bytes == pk.vk_bytes
                cproof, pos, _ = cp.prove(circ.instance, circ.witness, seed, rounds, pos0)
                assert cproof == gproof
                assert pos == rng.word_pos
            finally:
                cp.close()
            if log_n == 13:
                # sample_mask's first pass makes need + need / 8 + 1024 attempts; the proof's other draws are a few dozen
                # words, so more attempts than that plus a wide margin means the mask took a second pass
                need = 3 * n
                assert (rng.word_pos - pos0) // 8 > need + need // 8 + 1024 + 1000
        finally:
            pk.close()
    finally:
        srs.close()


# ---------------------------------------------------------------------------------------------------
# H. MSM digit recoding at every window width
# ---------------------------------------------------------------------------------------------------
def digit_patterns(curve, c):
    """Scalars aimed at msm_digits_kernel's signed-digit recoding at window width c."""
    r = curve.fr.p
    bits = curve.fr.bits
    W = (bits + 1 + c - 1) // c
    half, full = 1 << (c - 1), (1 << c) - 1
    below = (1 << (bits - 1)) - 1  # keeps a pattern < r, so that it reaches the kernel unreduced

    def every(*ws):
        return sum(ws[w % len(ws)] << (w * c) for w in range(W)) & below

    pats = [every(half), every(half + 1), every(full), every(half - 1), every(half + 1, half - 1), every(half, half + 1),
            every(full, 0), every(1, full), every(half + 1, full, half),
            r - 1, r - 2, 1 << (bits - 1), (1 << ((W - 1) * c)) - 1, (1 << ((W - 2) * c)) - 1, (1 << ((W - 1) * c)) % r,
            r - (1 << ((W - 2) * c)), half << ((W - 2) * c), (half + 1) << ((W - 2) * c), 0, 1, half, half + 1, full,
            int("55" * 32, 16) & below, int("aa" * 32, 16) & below, int("cc" * 32, 16) % r, int("33" * 32, 16) % r]
    return [v % r for v in pats]


_powers_cache = {}


def _key_powers(ctx, curve, n, beta):
    import b2m_testutil as util
    k = (curve.name, n, beta)
    if k not in _powers_cache:
        _powers_cache.clear()
        _powers_cache[k] = util.gpu_powers(ctx, curve, curve.g, beta, n)
    return _powers_cache[k]


@pytest.mark.parametrize("curve", CURVES, ids=lambda c: c.name)
@pytest.mark.parametrize("c", list(range(8, 25)))
def test_msm_digit_recoding(b2m_ctx, curve, c):
    """A 2^10-power key at window width c = 8..24: windows of 2^(c-1) (the digit stays positive), 2^(c-1) + 1 (it flips and
    carries), 2^c - 1 (carry chains, mag = 0 -> no digit), the carry out of the top window (at c = 15 and 17 on
    BLS12-381, 255 = 15 * 17, it survives only through the + 1 in W = (BITS + 1 + c - 1) / c), against the trapdoor."""
    import b2m_testutil as util
    from marlin_b200 import _lib
    L = _lib.lib()
    r = curve.fr.p
    n = 1 << 10
    beta = 0x3c5a7e91b2d4f60817293a4b5c6d7e8f % r
    rnd = random.Random(c * 3 + len(curve.name))
    srs = util.make_srs(b2m_ctx, curve, _key_powers(b2m_ctx, curve, n, beta), window_bits=c)
    try:
        assert L.b2m_srs_window_bits(srs) == c
        pats = digit_patterns(curve, c)
        tiled = [pats[i % len(pats)] for i in range(n)]
        mixed = [rnd.choice(pats) if rnd.randrange(2) else rnd.randrange(r) for _ in range(n - 3)]
        cases = [(0, pats), (n - len(pats), pats), (0, tiled), (3, mixed), (0, [rnd.randrange(r) for _ in range(64)]), (1, [pats[9]] * 5)]
        cases += [(i, [v]) for i, v in enumerate(pats[9:18])]  # r - 1 and the top-window values alone
        for off, sc in cases:
            assert util.srs_msm(srs, curve, off, sc) == util.trapdoor_msm(curve, curve.g, beta, off, sc), (c, off, len(sc))
    finally:
        L.b2m_srs_destroy(srs)


@pytest.mark.parametrize("curve", CURVES, ids=lambda c: c.name)
def test_msm_benchmark_width(b2m_ctx, monkeypatch, curve):
    """The benchmark's MSM shape with default knobs: a 2^21-power key (pick_window -> c = 20), an MSM over all 2^21
    scalars and one over a slice at a non-zero offset; on BLS12-381 both are above the 2^23-reference threshold of the
    batched-affine levels (13 * 2^21 and 13 * (2^20 + 1)), on BN254 the levels are off.  Random scalars plus the digit
    patterns of c = 20, against the trapdoor."""
    import b2m_testutil as util
    from marlin_b200 import _lib
    for k in list(os.environ):
        if k.startswith("B2M_MSM_"):
            monkeypatch.delenv(k)
    L = _lib.lib()
    r = curve.fr.p
    n = 1 << 21
    beta = 0x2f8a9b1c3d4e5f60718293a4b5c6d7e8f9 % r
    srs = util.make_srs(b2m_ctx, curve, _key_powers(b2m_ctx, curve, n, beta))
    try:
        c = L.b2m_srs_window_bits(srs)
        assert c == 20
        W = (curve.fr.bits + 1 + c - 1) // c
        bls = curve is BLS12_381
        assert L.b2m_srs_affine_levels(srs) == (3 if bls else 0)
        m = n // 2 + 1
        if bls:
            assert W * m > (1 << 23)
        rng = np.random.default_rng(20 + len(curve.name))
        raw = rng.integers(0, 1 << 63, size=(n, 4), dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=(n, 4), dtype=np.uint64)
        raw[:, 3] &= np.uint64((1 << (curve.fr.bits - 1 - 192)) - 1)  # < 2^(bits - 1) < r
        pats = digit_patterns(curve, c)
        idx = np.arange(0, n, 4099)[: 4 * len(pats)]
        raw[idx] = _lib.ints_to_limbs([pats[i % len(pats)] for i in range(len(idx))], 4)
        raw[: len(pats)] = _lib.ints_to_limbs(pats, 4)
        sc = _lib.limbs_to_ints(raw)

        def msm(off, arr):
            out = np.zeros(2 * curve.fq.limbs64, dtype=np.uint64)
            inf = ctypes.c_int(0)
            _lib.check(L.b2m_srs_msm(srs, off, _lib.ptr(np.ascontiguousarray(arr)), len(arr), _lib.ptr(out), ctypes.byref(inf)))
            return util.points_from_limbs(curve, out)[0]

        assert msm(0, raw) == util.trapdoor_msm(curve, curve.g, beta, 0, sc)
        assert msm(77, raw[:m]) == util.trapdoor_msm(curve, curve.g, beta, 77, sc[:m])
    finally:
        L.b2m_srs_destroy(srs)
