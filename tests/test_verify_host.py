"""CPU: the verifier's host-compiled pieces -- the compressed-G1 decoder the decode kernel runs (csrc/g1_decode.cuh) and the
pairing product check (csrc/pairing_host.hpp) -- against the oracle (oracle/marlin.py::_g1_decompress, oracle/pairing.py)."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

from oracle import ec, pairing as opairing
from oracle import marlin as omarlin
from oracle import transcript as T
from oracle.params import BLS12_381, BN254

HERE = os.path.dirname(os.path.abspath(__file__))
CURVES = list(enumerate([BLS12_381, BN254]))
IDS = lambda x: getattr(x, "name", x)  # noqa: E731


@pytest.fixture(scope="module")
def hostlib(tmp_path_factory):
    src = os.path.join(HERE, "host", "verify_host_shim.cpp")
    so = str(tmp_path_factory.mktemp("verify_host") / "libverify_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-DB2M_HOST_LIGHT_INLINE", "-shared", "-fPIC", "-x", "c++", src, "-o", so])
    return ctypes.CDLL(so)


def n32(ci):
    return 12 if ci == 0 else 8


def pack_g1(curve, ci, pts):
    out = []
    for P in pts:
        if P is None:
            out += [0] * (2 * n32(ci))
            continue
        for v in P:
            m = curve.fq.to_mont(v)
            out += [(m >> (32 * i)) & 0xffffffff for i in range(n32(ci))]
    return np.array(out, dtype=np.uint32)


def unpack_g1(curve, ci, arr):
    n = n32(ci)
    x = sum(int(arr[i]) << (32 * i) for i in range(n))
    y = sum(int(arr[n + i]) << (32 * i) for i in range(n))
    return None if x == 0 and y == 0 else (curve.fq.from_mont(x), curve.fq.from_mont(y))


def g2_bytes(ci, scalars):
    """k * (standard G2 generator) as ark-serialize uncompressed bytes (b2m_g2_scalar_muls runs on the host)."""
    from marlin_b200 import _lib
    nb = 4 * (48 if ci == 0 else 32)
    sc = _lib.ints_to_limbs(list(scalars), 4)
    out = np.zeros(nb * len(scalars), dtype=np.uint8)
    _lib.check(_lib.lib().b2m_g2_scalar_muls(ci, None, _lib.ptr(sc), len(scalars), _lib.ptr(out)))
    return out.tobytes()


def g2_to_oracle(curve, blob):
    nq = curve.fq.nbytes
    v = [int.from_bytes(blob[k * nq:(k + 1) * nq], "little") for k in range(4)]
    v[3] &= ~(0xc0 << (8 * (nq - 1)))
    return opairing.for_curve(curve).untwist((v[0], v[1]), (v[2], v[3]))


def decode(hostlib, ci, curve, blobs):
    n = len(blobs)
    out = np.zeros(n * 2 * n32(ci), dtype=np.uint32)
    st = np.zeros(n, dtype=np.int32)
    data = np.frombuffer(b"".join(blobs), dtype=np.uint8)
    hostlib.g1_decode_host(ci, data.ctypes.data_as(ctypes.c_void_p), n, out.ctypes.data_as(ctypes.c_void_p), st.ctypes.data_as(ctypes.c_void_p))
    return [(int(st[i]), unpack_g1(curve, ci, out[i * 2 * n32(ci):(i + 1) * 2 * n32(ci)])) for i in range(n)]


@pytest.mark.parametrize("ci,curve", CURVES, ids=IDS)
def test_g1_decode_matches_oracle(hostlib, ci, curve):
    rnd = random.Random(40 + ci)
    fq = curve.fq
    pts = [ec.scalar_mul(curve, rnd.randrange(1, curve.fr.p), curve.g) for _ in range(24)]
    pts.append(ec.affine_neg(curve, pts[0]))  # both signs of one x
    blobs = [T.g1_compressed(curve, P) for P in pts] + [T.g1_compressed(curve, None)]
    got = decode(hostlib, ci, curve, blobs)
    assert {P[1] > (fq.p - P[1]) for P in pts} == {True, False}
    for (st, P), blob, want in zip(got, blobs, pts + [None]):
        assert st == 0 and P == want == omarlin._g1_decompress(curve, blob)

    def enc(x, flags=0):
        b = bytearray(x.to_bytes(fq.nbytes, "little"))
        b[-1] |= flags
        return bytes(b)

    # x >= p (with either sign flag), both flag bits set
    assert [s for s, _ in decode(hostlib, ci, curve, [enc(fq.p), enc(fq.p + 5, 0x80)])] == [2, 2]
    both = bytearray(blobs[0])
    both[-1] |= 0xc0
    assert decode(hostlib, ci, curve, [bytes(both)])[0][0] == 1
    # x with no square root of x^3 + b
    x = next(x for x in range(1, 1000) if pow((x ** 3 + curve.b) % fq.p, (fq.p - 1) // 2, fq.p) == fq.p - 1)
    assert decode(hostlib, ci, curve, [enc(x)])[0][0] == 3
    with pytest.raises(ValueError):
        omarlin._g1_decompress(curve, enc(x))


def test_g1_decode_rejects_points_outside_the_bls_subgroup(hostlib):
    """A BLS12-381 curve point whose cofactor was not cleared is on the curve but not in G1: rejected."""
    curve, fq = BLS12_381, BLS12_381.fq
    x = next(x for x in range(1, 1000) if pow((x ** 3 + curve.b) % fq.p, (fq.p - 1) // 2, fq.p) == 1)
    y = pow((x ** 3 + curve.b) % fq.p, (fq.p + 1) // 4, fq.p)
    assert ec.affine_add(curve, ec.scalar_mul(curve, curve.fr.p - 1, (x, y)), (x, y)) is not None  # r * P != O
    for P in ((x, y), (x, fq.p - y)):
        assert omarlin._g1_decompress(curve, T.g1_compressed(curve, P)) == P  # the oracle has no subgroup check
        assert decode(hostlib, 0, curve, [T.g1_compressed(curve, P)])[0][0] == 4
    # BN254 G1 has cofactor 1: every curve point is in the group
    bn = BN254
    x = next(x for x in range(1, 1000) if pow((x ** 3 + bn.b) % bn.fq.p, (bn.fq.p - 1) // 2, bn.fq.p) == 1)
    y = pow((x ** 3 + bn.b) % bn.fq.p, (bn.fq.p + 1) // 4, bn.fq.p)
    assert decode(hostlib, 1, bn, [T.g1_compressed(bn, (x, y))])[0] == (0, (x, y))


def pairing_value(hostlib, ci, curve, P, qbytes):
    out = np.zeros(12 * n32(ci), dtype=np.uint32)
    pts = pack_g1(curve, ci, [P])
    ok = ctypes.c_int(0)
    assert hostlib.pairing_host(ci, 1, 1, pts.ctypes.data_as(ctypes.c_void_p), qbytes, ctypes.byref(ok), out.ctypes.data_as(ctypes.c_void_p)) == 0
    n = n32(ci)
    return opairing.for_curve(curve).Fq12([curve.fq.from_mont(sum(int(out[k * n + i]) << (32 * i) for i in range(n))) for k in range(12)])


def product_is_one(hostlib, ci, curve, pts, qbytes):
    ok = ctypes.c_int(-1)
    arr = pack_g1(curve, ci, pts)
    rc = hostlib.pairing_host(ci, 0, len(pts), arr.ctypes.data_as(ctypes.c_void_p), qbytes, ctypes.byref(ok), None)
    assert rc == 0
    return bool(ok.value)


@pytest.mark.parametrize("ci,curve", CURVES, ids=IDS)
def test_pairing_bilinear_nondegenerate_and_equal_to_the_oracle(hostlib, ci, curve):
    rnd = random.Random(60 + ci)
    r = curve.fr.p
    pg = opairing.for_curve(curve)
    a, b = rnd.randrange(1, r), rnd.randrange(1, r)
    q1, qb = g2_bytes(ci, [1]), g2_bytes(ci, [b])
    e = pairing_value(hostlib, ci, curve, curve.g, q1)
    assert e != pg.Fq12.one()                                      # non-degenerate
    assert e.pow(r) == pg.Fq12.one()                               # e(P, Q)^r = 1
    assert e == pg.pairing(curve.g, g2_to_oracle(curve, q1))       # the oracle's reduced Tate pairing, value for value
    e_ab = pairing_value(hostlib, ci, curve, ec.scalar_mul(curve, a, curve.g), qb)
    assert e_ab == e.pow(a * b % r)                                # bilinear


@pytest.mark.parametrize("ci,curve", CURVES, ids=IDS)
def test_pairing_product_agrees_with_the_oracle(hostlib, ci, curve):
    """e(aG, bH) e(-cG, dH) e(xG, yH) == 1 iff ab - cd + xy = 0 (mod r), decided like oracle/pairing.py decides it."""
    rnd = random.Random(70 + ci)
    r = curve.fr.p
    pg = opairing.for_curve(curve)
    for accept in (True, False, True, False):
        a, b, c, d, y = (rnd.randrange(1, r) for _ in range(5))
        x = (c * d - a * b) * pow(y, -1, r) % r
        if not accept:
            x = (x + rnd.randrange(1, r)) % r
        pts = [ec.scalar_mul(curve, a, curve.g), ec.affine_neg(curve, ec.scalar_mul(curve, c, curve.g)), ec.scalar_mul(curve, x, curve.g)]
        qs = g2_bytes(ci, [b, d, y])
        got = product_is_one(hostlib, ci, curve, pts, qs)
        assert got == accept
        nq = len(qs) // 3
        assert got == pg.pairing_product_is_one([(P, g2_to_oracle(curve, qs[i * nq:(i + 1) * nq])) for i, P in enumerate(pts)])
    # infinity on the G1 side contributes 1
    assert product_is_one(hostlib, ci, curve, [None, curve.g, ec.affine_neg(curve, curve.g)], g2_bytes(ci, [3, 5, 5]))


@pytest.mark.parametrize("ci,curve", CURVES, ids=IDS)
def test_pairing_rejects_g2_points_off_the_curve(hostlib, ci, curve):
    q = bytearray(g2_bytes(ci, [7]))
    q[0] ^= 1
    arr = pack_g1(curve, ci, [curve.g])
    ok = ctypes.c_int(0)
    assert hostlib.pairing_host(ci, 0, 1, arr.ctypes.data_as(ctypes.c_void_p), bytes(q), ctypes.byref(ok), None) == -1
