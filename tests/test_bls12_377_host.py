"""CPU: the BLS12-377 instantiation of the device arithmetic compiled for the host (tests/host/bls12_377_host_shim.cpp),
checked against Python integers and the oracle: the constants re-derived from the curve parameter u, Fr / Fq at their edges,
Tonelli-Shanks, the beta = 5 Fq2, G1 / G2 decoding, the endomorphism subgroup test and the host pairing."""
import ctypes
import os
import random
import subprocess

import pytest

import bls12_377_oracle as B
from marlin_b200 import _lib, fields
from oracle import ec

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "marlin_b200", "csrc")
Q, R, U = B.Q_MOD, B.R_MOD, B.U
CURVE = B.BLS12_377
NQ, NR = 12, 8


@pytest.fixture(scope="module")
def hostlib(tmp_path_factory):
    src = os.path.join(HERE, "host", "bls12_377_host_shim.cpp")
    so = str(tmp_path_factory.mktemp("bls377") / "libbls377_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-DB2M_HOST_LIGHT_INLINE", "-shared", "-fPIC", "-x", "c++", src, "-o", so])
    return ctypes.CDLL(so)


def limbs(x, n):
    return (ctypes.c_uint32 * n)(*[(x >> (32 * i)) & 0xffffffff for i in range(n)])


def unlimbs(a, off=0, n=NQ):
    return sum(int(a[off + i]) << (32 * i) for i in range(n))


def field_op(lib, field, which, a, b=0):
    n = NR if field == 0 else NQ
    r = (ctypes.c_uint32 * n)()
    ok = lib.field_op(field, which, limbs(a, n), limbs(b, n), r)
    return unlimbs(r, n=n), ok


def fq2_op(lib, which, a, b=(0, 0)):
    r = (ctypes.c_uint32 * (2 * NQ))()
    ok = lib.fq2_op(which, limbs(a[0] | (a[1] << (32 * NQ)), 2 * NQ), limbs(b[0] | (b[1] << (32 * NQ)), 2 * NQ), r)
    return (unlimbs(r, 0), unlimbs(r, NQ)), ok


def fq_bytes(x):
    return x.to_bytes(48, "little")


def g1_compressed(P):
    if P is None:
        return bytes(47) + b"\x40"
    b = bytearray(fq_bytes(P[0]))
    if P[1] > (Q - 1) // 2:
        b[47] |= 0x80
    return bytes(b)


def g1_uncompressed(P):
    if P is None:
        return bytes(95) + b"\x40"
    return fq_bytes(P[0]) + fq_bytes(P[1])


def fq2_gt_neg(y):
    return y[1] > (Q - 1) // 2 if y[1] else y[0] > (Q - 1) // 2


def g2_uncompressed(P):
    (x0, x1), (y0, y1) = P
    return fq_bytes(x0) + fq_bytes(x1) + fq_bytes(y0) + fq_bytes(y1)


def g2_compressed(P):
    x, y = P
    b = bytearray(fq_bytes(x[0]) + fq_bytes(x[1]))
    if fq2_gt_neg(y):
        b[95] |= 0x80
    return bytes(b)


def decode_g1(lib, blobs, compressed):
    n = len(blobs)
    out = (ctypes.c_uint32 * (2 * NQ * n))()
    st = (ctypes.c_int * n)()
    lib.g1_decode_host(b"".join(blobs), n, int(compressed), out, st)
    pts = []
    for i in range(n):
        x, y = unlimbs(out, 2 * NQ * i), unlimbs(out, 2 * NQ * i + NQ)
        pts.append(None if x == 0 and y == 0 else (x, y))
    return pts, list(st)


def decode_g2(lib, blobs, compressed):
    n = len(blobs)
    out = ctypes.create_string_buffer(4 * 48 * n)
    st = (ctypes.c_int * n)()
    lib.g2_decode_host(b"".join(blobs), n, int(compressed), out, st)
    return [out.raw[192 * i:192 * (i + 1)] for i in range(n)], list(st)


def raw_curve_point(rnd):
    """a uniformly chosen point of E(Fq) (almost surely outside G1)"""
    while True:
        x = rnd.randrange(Q)
        y = B.fq_sqrt(x ** 3 + 1)
        if y is not None and y:
            return (x, y)


def g1_mul(k, P):
    return ec.scalar_mul(CURVE, k, P) if k % R else _full_mul(k, P)


def _full_mul(k, P):
    acc = None
    while k:
        if k & 1:
            acc = ec.affine_add(CURVE, acc, P)
        P, k = ec.affine_add(CURVE, P, P), k >> 1
    return acc


# ---- constants ---------------------------------------------------------------------------------------------------------

def test_constants_rederived_from_u():
    assert R == U ** 4 - U ** 2 + 1 and Q == (U - 1) ** 2 * R // 3 + U
    assert R.bit_length() == 253 and Q.bit_length() == 377
    assert B.FR.two_adicity == 47 and B.FQ.two_adicity == 46 and Q % 3 == 1
    assert fields.FR_MODULUS[_lib.CURVE_BLS12_377] == R and fields.FQ_MODULUS[_lib.CURVE_BLS12_377] == Q
    assert fields.CURVE_IDS["bls12_377"] == 2 and _lib.LIMBS[2] == (4, 6)
    # Fr generator 22: a non-residue whose two-adic root has exact order 2^47 (coset shift of the NTT)
    root = pow(22, (R - 1) >> 47, R)
    assert pow(root, 1 << 46, R) == R - 1
    # G1: generator on y^2 = x^3 + 1, of order r, and phi(G) = -u^2 G for omega = 2^((q - 1) / 3) only
    G = CURVE.g
    assert fields.G1_GENERATOR[2] == G and ec.on_curve(CURVE, G)
    assert _full_mul(R, G) is None
    u2g = _full_mul(U * U % R, G)
    assert (B.OMEGA * G[0] % Q, G[1]) == ec.affine_neg(CURVE, u2g)
    assert (B.OMEGA * B.OMEGA * G[0] % Q, G[1]) != ec.affine_neg(CURVE, u2g)
    # twist: b' = 1 / u with u^2 = -5; the G2 generator lies on it and has order r
    assert B.fq2_mul(B.B_TWIST, (0, 1)) == (1, 0)
    x, y = (B.G2_GENERATOR[0], B.G2_GENERATOR[1]), (B.G2_GENERATOR[2], B.G2_GENERATOR[3])
    assert B.g2_on_twist(x, y) and B.g2_mul(R, (x, y)) is None
    # the generated device parameters match
    text = open(os.path.join(CSRC, "field_params.h")).read()
    for name, p, tw in (("Bls377FrParams", R, 47), ("Bls377FqParams", Q, 46)):
        blk = text[text.index("struct " + name):]
        blk = blk[:blk.index("};")]
        assert f"TWO_ADICITY = {tw};" in blk
        assert ", ".join("0x%08xu" % ((p >> (32 * i)) & 0xffffffff) for i in range(NR if p == R else NQ)) in blk


# ---- fields ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("field", [0, 1], ids=["fr", "fq"])
def test_field_mul_inverse_edges(hostlib, field):
    p = R if field == 0 else Q
    n = NR if field == 0 else NQ
    rnd = random.Random(field)
    top = [(1 << (p.bit_length() - 1)) + rnd.randrange(1 << 64) for _ in range(4)]
    vals = [0, 1, 2, p - 1, p - 2, (p - 1) // 2, (p + 1) // 2, (1 << (32 * (n - 1))) % p] + top + [rnd.randrange(p) for _ in range(40)]
    for a in vals:
        for b in vals[:12]:
            assert field_op(hostlib, field, 0, a, b)[0] == a * b % p
            assert field_op(hostlib, field, 1, a, b)[0] == (a + b) % p
            assert field_op(hostlib, field, 2, a, b)[0] == (a - b) % p
        inv = pow(a, -1, p) if a else 0
        assert field_op(hostlib, field, 3, a)[0] == inv
        assert field_op(hostlib, field, 4, a)[0] == inv


def test_tonelli_shanks(hostlib):
    rnd = random.Random(7)
    cases = [0, 1, Q - 1, 4, 15] + [rnd.randrange(Q) ** 2 % Q for _ in range(40)] + [rnd.randrange(Q) for _ in range(40)]
    # squares whose a^t has high 2-power order (many Tonelli-Shanks rounds)
    root = pow(15, (Q - 1) >> 46, Q)
    cases += [pow(root, 2 * k + 1, Q) ** 2 % Q for k in range(4)] + [pow(root, 1 << 44, Q)]
    for a in cases:
        s, ok = field_op(hostlib, 1, 5, a)
        square = a == 0 or pow(a, (Q - 1) // 2, Q) == 1
        assert ok == int(square), hex(a)
        if square:
            assert s * s % Q == a
    assert field_op(hostlib, 1, 5, 15)[1] == 0  # the generator is a non-residue


def test_fq2_beta5(hostlib):
    rnd = random.Random(11)
    vals = [(0, 0), (1, 0), (0, 1), (Q - 1, Q - 1), (5, 0), (0, Q - 1)] + [(rnd.randrange(Q), rnd.randrange(Q)) for _ in range(20)]
    for a in vals:
        for b in vals[:8]:
            assert fq2_op(hostlib, 0, a, b)[0] == B.fq2_mul(a, b)
        if a != (0, 0):
            assert fq2_op(hostlib, 1, a)[0] == B.fq2_inv(a)
    assert fq2_op(hostlib, 0, (0, 1), (0, 1))[0] == (Q - 5, 0)  # u^2 = -5
    sq = [B.fq2_mul(a, a) for a in vals] + [(Q - 5, 0), (rnd.randrange(Q) ** 2 % Q, 0), (Q - 1, 0)]
    nonsq = []
    while len(nonsq) < 8:
        a = (rnd.randrange(Q), rnd.randrange(Q))
        if B.fq2_sqrt(a) is None:
            nonsq.append(a)
    for a in sq + nonsq:
        s, ok = fq2_op(hostlib, 2, a)
        expect = B.fq2_sqrt(a) is not None
        assert ok == int(expect), a
        if ok:
            assert B.fq2_mul(s, s) == (a[0] % Q, a[1] % Q)


# ---- points ------------------------------------------------------------------------------------------------------------

def test_g1_decode_against_oracle(hostlib):
    rnd = random.Random(3)
    pts = [CURVE.g] + [g1_mul(rnd.randrange(1, R), CURVE.g) for _ in range(12)] + [None]
    for compressed in (True, False):
        enc = g1_compressed if compressed else g1_uncompressed
        got, st = decode_g1(hostlib, [enc(P) for P in pts], compressed)
        assert st == [0] * len(pts) and got == pts
    # rejections: both flags, x >= q, off the curve, cofactor torsion, (0, +-1)
    raw = raw_curve_point(rnd)
    tors = _full_mul(R, raw)
    assert tors is not None
    x_off = next(x for x in range(2, 100) if B.fq_sqrt(x ** 3 + 1) is None)
    bad = [bytes(47) + b"\xc0", fq_bytes(Q), fq_bytes(x_off), g1_compressed(tors), g1_compressed(raw), g1_compressed((0, 1)),
           g1_compressed((0, Q - 1))]
    _, st = decode_g1(hostlib, bad, True)
    assert st == [1, 2, 3, 4, 4, 4, 4]
    badu = [g1_uncompressed(tors), g1_uncompressed((0, 1)), fq_bytes(1) + fq_bytes(1), fq_bytes(0) + fq_bytes(Q)]
    _, st = decode_g1(hostlib, badu, False)
    assert st == [4, 4, 3, 5]


def test_g1_endomorphism_subgroup_test(hostlib):
    rnd = random.Random(5)
    sub = [g1_mul(rnd.randrange(1, R), CURVE.g) for _ in range(6)]
    raw = [raw_curve_point(rnd) for _ in range(6)]
    tors = [_full_mul(R, P) for P in raw]
    sums = [ec.affine_add(CURVE, s, t) for s, t in zip(sub, tors)]
    small = [(0, 1), (0, Q - 1)]
    pts = sub + raw + [t for t in tors if t] + [s for s in sums if s] + small
    arr = (ctypes.c_uint32 * (2 * NQ * len(pts)))()
    for i, P in enumerate(pts):
        for k, c in enumerate(P):
            for j in range(NQ):
                arr[2 * NQ * i + NQ * k + j] = (c >> (32 * j)) & 0xffffffff
    out = (ctypes.c_int * (2 * len(pts)))()
    hostlib.g1_subgroup_host(arr, len(pts), out)
    for i, P in enumerate(pts):
        assert out[2 * i] == out[2 * i + 1], P
        assert out[2 * i] == int(i < len(sub)), P


def test_g2_decode_against_oracle(hostlib):
    rnd = random.Random(9)
    gen = ((B.G2_GENERATOR[0], B.G2_GENERATOR[1]), (B.G2_GENERATOR[2], B.G2_GENERATOR[3]))
    pts = [gen] + [B.g2_mul(rnd.randrange(1, R), gen) for _ in range(3)]
    for compressed in (True, False):
        enc = g2_compressed if compressed else g2_uncompressed
        got, st = decode_g2(hostlib, [enc(P) for P in pts], compressed)
        assert st == [0] * len(pts)
        assert got == [g2_uncompressed(P) for P in pts]
    # a point on the twist outside the order-r subgroup, a non-twist x, and x.c1 >= q
    while True:
        x = (rnd.randrange(Q), rnd.randrange(Q))
        y = B.fq2_sqrt(B.fq2_add(B.fq2_mul(B.fq2_mul(x, x), x), B.B_TWIST))
        if y is not None:
            break
    while True:
        xn = (rnd.randrange(Q), rnd.randrange(Q))
        if B.fq2_sqrt(B.fq2_add(B.fq2_mul(B.fq2_mul(xn, xn), xn), B.B_TWIST)) is None:
            break
    _, st = decode_g2(hostlib, [g2_compressed((x, y)), fq_bytes(xn[0]) + fq_bytes(xn[1]), fq_bytes(1) + fq_bytes(Q)], True)
    assert st == [4, 3, 2]


# ---- pairing -----------------------------------------------------------------------------------------------------------

def host_pairing(lib, P, Qg2):
    pts = limbs((P[0] | (P[1] << (32 * NQ))) if P else 0, 2 * NQ)
    out = (ctypes.c_uint32 * (12 * NQ))()
    ok = ctypes.c_int()
    assert lib.pairing_host(1, 1, pts, g2_uncompressed(Qg2), ctypes.byref(ok), out) == 0
    return [unlimbs(out, NQ * k) for k in range(12)]


def test_host_pairing_matches_oracle_and_is_bilinear(hostlib):
    eng = B.register()
    rnd = random.Random(13)
    gen = ((B.G2_GENERATOR[0], B.G2_GENERATOR[1]), (B.G2_GENERATOR[2], B.G2_GENERATOR[3]))
    P = g1_mul(rnd.randrange(1, R), CURVE.g)
    e = host_pairing(hostlib, P, gen)
    assert e == eng.pairing(P, eng.untwist(*gen)).c
    assert e != eng.Fq12.one().c  # non-degenerate
    a, b = rnd.randrange(1, R), rnd.randrange(1, R)
    eab = host_pairing(hostlib, g1_mul(a, P), B.g2_mul(b, gen))
    assert eab == eng.Fq12(e).pow(a * b % R).c
    # product check: e(aP, Q) e(-P, aQ) == 1, and not with a wrong scalar
    aP, negP = g1_mul(a, P), ec.affine_neg(CURVE, P)
    pts = limbs(sum((c << (32 * NQ * k)) for k, c in enumerate([aP[0], aP[1], negP[0], negP[1]])), 4 * NQ)
    ok = ctypes.c_int()
    g2 = g2_uncompressed(gen) + g2_uncompressed(B.g2_mul(a, gen))
    assert hostlib.pairing_host(0, 2, pts, g2, ctypes.byref(ok), None) == 0 and ok.value == 1
    g2bad = g2_uncompressed(gen) + g2_uncompressed(B.g2_mul(a + 1, gen))
    assert hostlib.pairing_host(0, 2, pts, g2bad, ctypes.byref(ok), None) == 0 and ok.value == 0
