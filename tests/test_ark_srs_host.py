"""CPU: the SRS loader's shared point code compiled for the host (csrc/g1_decode.cuh, csrc/g2_decode.cuh, the bodies of the
decode kernels) against the Python oracle -- both curves, both groups, both forms, every rejection class, the BLS12-381
endomorphism subgroup test against r * P = O -- and the framing checks of marlin_b200.srsfile.read_ark."""
import ctypes
import os
import random
import struct
import subprocess

import numpy as np
import pytest

from oracle import ec
from oracle import transcript as T
from oracle.params import BLS12_381, BN254

import ark_srs_oracle as ao

HERE = os.path.dirname(os.path.abspath(__file__))
CURVES = list(enumerate([BLS12_381, BN254]))
IDS = lambda x: getattr(x, "name", x)  # noqa: E731
OK, BAD_FLAGS, X_NC, NOT_ON_CURVE, NOT_IN_SUBGROUP, Y_NC = range(6)


@pytest.fixture(scope="module")
def hostlib(tmp_path_factory):
    src = os.path.join(HERE, "host", "ark_points_host_shim.cpp")
    so = str(tmp_path_factory.mktemp("ark_host") / "libark_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-DB2M_HOST_LIGHT_INLINE", "-shared", "-fPIC", "-x", "c++", src, "-o", so])
    return ctypes.CDLL(so)


def n32(ci):
    return 12 if ci == 0 else 8


def vp(a):
    return a.ctypes.data_as(ctypes.c_void_p)


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


def g1_decode(lib, ci, curve, blobs, compressed):
    n = len(blobs)
    out = np.zeros(n * 2 * n32(ci), dtype=np.uint32)
    st = np.zeros(n, dtype=np.int32)
    data = np.frombuffer(b"".join(blobs), dtype=np.uint8).copy()
    lib.g1_decode_ark_host(ci, vp(data), n, int(compressed), vp(out), vp(st))
    return [(int(st[i]), unpack_g1(curve, ci, out[i * 2 * n32(ci):(i + 1) * 2 * n32(ci)])) for i in range(n)]


def g2_decode(lib, ci, blobs, compressed):
    n = len(blobs)
    nb = 4 * n32(ci) * 4
    out = np.zeros(n * nb, dtype=np.uint8)
    st = np.zeros(n, dtype=np.int32)
    data = np.frombuffer(b"".join(blobs), dtype=np.uint8).copy()
    lib.g2_decode_ark_host(ci, vp(data), n, int(compressed), vp(out), vp(st))
    raw = out.tobytes()
    return [(int(st[i]), raw[i * nb:(i + 1) * nb]) for i in range(n)]


def raw_g1(curve, start=1):
    """a curve point with the cofactor not cleared"""
    fq = curve.fq
    x = next(x for x in range(start, start + 1000) if pow((x ** 3 + curve.b) % fq.p, (fq.p - 1) // 2, fq.p) == 1)
    return (x, pow((x ** 3 + curve.b) % fq.p, (fq.p + 1) // 4, fq.p))


def enc(fq, x, flags=0):
    b = bytearray(x.to_bytes(fq.nbytes, "little"))
    b[-1] |= flags
    return bytes(b)


@pytest.mark.parametrize("compressed", [True, False], ids=["compressed", "uncompressed"])
@pytest.mark.parametrize("ci,curve", CURVES, ids=IDS)
def test_g1_decoders_match_the_oracle_and_compress_back(hostlib, ci, curve, compressed):
    rnd = random.Random(10 + ci)
    pts = [ec.scalar_mul(curve, rnd.randrange(1, curve.fr.p), curve.g) for _ in range(16)]
    pts += [ec.affine_neg(curve, pts[0]), None]
    blobs = [ao.g1_bytes(curve, P, compressed) for P in pts]
    assert g1_decode(hostlib, ci, curve, blobs, compressed) == [(OK, P) for P in pts]
    comp = np.zeros(len(pts) * curve.fq.nbytes, dtype=np.uint8)
    hostlib.g1_compress_host(ci, vp(pack_g1(curve, ci, pts)), len(pts), vp(comp))
    assert comp.tobytes() == b"".join(T.g1_compressed(curve, P) for P in pts)


@pytest.mark.parametrize("ci,curve", CURVES, ids=IDS)
def test_g1_decoders_reject_every_invalid_class(hostlib, ci, curve):
    fq = curve.fq
    G = curve.g
    good_c, good_u = T.g1_compressed(curve, G), ao.g1_uncompressed(curve, G)
    both_c, both_u = bytearray(good_c), bytearray(good_u)
    both_c[-1] |= 0xc0
    both_u[-1] |= 0xc0
    x_nosqrt = next(x for x in range(1, 1000) if pow((x ** 3 + curve.b) % fq.p, (fq.p - 1) // 2, fq.p) == fq.p - 1)
    comp = [bytes(both_c), enc(fq, fq.p), enc(fq, fq.p + 3, 0x80), enc(fq, x_nosqrt)]
    assert [s for s, _ in g1_decode(hostlib, ci, curve, comp, True)] == [BAD_FLAGS, X_NC, X_NC, NOT_ON_CURVE]
    unc = [bytes(both_u), enc(fq, fq.p) + enc(fq, G[1]), enc(fq, G[0]) + enc(fq, fq.p), enc(fq, G[0]) + enc(fq, G[1] + 1),
           enc(fq, G[0]) + enc(fq, fq.p + 1, 0x40)]
    assert [s for s, _ in g1_decode(hostlib, ci, curve, unc, False)] == [BAD_FLAGS, X_NC, Y_NC, NOT_ON_CURVE, Y_NC]
    R = raw_g1(curve)
    got = [s for s, _ in g1_decode(hostlib, ci, curve, [T.g1_compressed(curve, R)], True) + g1_decode(hostlib, ci, curve, [ao.g1_uncompressed(curve, R)], False)]
    assert got == ([NOT_IN_SUBGROUP] * 2 if ci == 0 else [OK] * 2)  # BN254 G1 has cofactor 1


def test_bls_endomorphism_subgroup_test_equals_r_times_p(hostlib):
    """phi(P) == -u^2 P agrees with r * P == O on subgroup points, raw curve points, pure torsion points r * Q and sums of
    subgroup and torsion points."""
    curve, r = BLS12_381, BLS12_381.fr.p
    rnd = random.Random(5)
    sub = [ec.scalar_mul(curve, rnd.randrange(1, r), curve.g) for _ in range(6)]
    raws = [raw_g1(curve, s) for s in (1, 50, 400, 1000, 7000, 33333)]

    def mul(k, P):  # k * P without reducing k mod r
        acc = None
        for bit in bin(k)[2:]:
            acc = ec.affine_add(curve, acc, acc)
            if bit == "1":
                acc = ec.affine_add(curve, acc, P)
        return acc
    tors = [mul(r, Q) for Q in raws]
    assert all(t is not None for t in tors)
    tors += [mul(3 * r, Q) for Q in raws[:2]] + [mul(0x396c8c005555e1568c00aaab0000aaab // 3 * r, raws[0])]  # smaller torsion orders
    tors = [t for t in tors if t is not None]
    sums = [ec.affine_add(curve, s, t) for s, t in zip(sub, tors)]
    pts = sub + raws + tors + sums
    out = np.zeros(2 * len(pts), dtype=np.int32)
    hostlib.g1_subgroup_host(0, vp(pack_g1(curve, 0, pts)), len(pts), vp(out))
    endo, by_r = out[0::2].tolist(), out[1::2].tolist()
    assert endo == by_r
    assert by_r == [1] * len(sub) + [0] * (len(pts) - len(sub))


@pytest.mark.parametrize("compressed", [True, False], ids=["compressed", "uncompressed"])
@pytest.mark.parametrize("ci,curve", CURVES, ids=IDS)
def test_g2_decoders_match_the_oracle_and_compress_back(hostlib, ci, curve, compressed):
    g2 = ao.G2(curve)
    rnd = random.Random(20 + ci)
    pts = [g2.smul(rnd.randrange(1, curve.fr.p), g2.gen) for _ in range(4)]
    pts += [g2.neg(pts[0]), None]
    assert {g2.larger(P[1]) for P in pts[:5]} == {True, False}
    enc2 = g2.compressed if compressed else g2.uncompressed
    got = g2_decode(hostlib, ci, [enc2(P) for P in pts], compressed)
    assert got == [(OK, g2.uncompressed(P)) for P in pts]
    for P in pts:
        assert g2.decompress(g2.compressed(P)) == P
    unc = np.frombuffer(b"".join(g2.uncompressed(P) for P in pts), dtype=np.uint8).copy()
    comp = np.zeros(len(pts) * 2 * curve.fq.nbytes, dtype=np.uint8)
    hostlib.g2_compress_host(ci, vp(unc), len(pts), vp(comp))
    assert comp.tobytes() == b"".join(g2.compressed(P) for P in pts)


@pytest.mark.parametrize("ci,curve", CURVES, ids=IDS)
def test_g2_decoders_reject_every_invalid_class(hostlib, ci, curve):
    g2, fq = ao.G2(curve), curve.fq
    nb = fq.nbytes
    G = g2.gen
    good_c, good_u = g2.compressed(G), g2.uncompressed(G)
    both_c, both_u = bytearray(good_c), bytearray(good_u)
    both_c[-1] |= 0xc0
    both_u[-1] |= 0xc0
    big = enc(fq, fq.p)
    x_bad = next(k for k in range(1000) if g2.eng._fq2_sqrt(g2.rhs((k, 1))) is None)
    comp = [bytes(both_c), big + good_c[nb:], good_c[:nb] + enc(fq, fq.p, 0x80), enc(fq, x_bad) + enc(fq, 1)]
    assert [s for s, _ in g2_decode(hostlib, ci, comp, True)] == [BAD_FLAGS, X_NC, X_NC, NOT_ON_CURVE]
    y_off = bytearray(good_u)
    y_off[2 * nb] ^= 1
    unc = [bytes(both_u), big + good_u[nb:], good_u[:2 * nb] + big + good_u[3 * nb:], good_u[:3 * nb] + enc(fq, fq.p + 1), bytes(y_off)]
    assert [s for s, _ in g2_decode(hostlib, ci, unc, False)] == [BAD_FLAGS, X_NC, Y_NC, Y_NC, NOT_ON_CURVE]
    R = g2.raw_point()
    assert g2.smul(curve.fr.p, R) is not None  # on the twist, outside the order-r subgroup
    assert [s for s, _ in g2_decode(hostlib, ci, [g2.compressed(R)], True)] == [NOT_IN_SUBGROUP]
    assert [s for s, _ in g2_decode(hostlib, ci, [g2.uncompressed(R)], False)] == [NOT_IN_SUBGROUP]


# ---- srsfile.read_ark framing ---------------------------------------------------------------------------------------------------
def small_file(tmp_path, compressed=True, D=3):
    blob, pts = ao.kzg10_setup(BLS12_381, D, 0x1234567, 7, True, compressed)
    path = os.path.join(tmp_path, "srs.bin")
    with open(path, "wb") as f:
        f.write(blob)
    return path, blob, pts


@pytest.mark.parametrize("compressed", [True, False], ids=["compressed", "uncompressed"])
def test_read_ark_parses_and_write_ark_reproduces(tmp_path, compressed):
    from marlin_b200 import srsfile
    path, blob, pts = small_file(tmp_path, compressed)
    d = srsfile.read_ark(path, 0, compressed)
    g1, g2 = srsfile.point_sizes(0, compressed)
    assert d["powers"].shape == (4, g1) and d["gamma_keys"].tolist() == list(range(5)) and d["neg_keys"].tolist() == list(range(4))
    assert d["gamma"].shape == (5, g1) and d["neg"].shape == (4, g2) and d["h"].shape == (g2,)
    out = os.path.join(tmp_path, "again.bin")
    srsfile.write_ark(out, 0, compressed, d["powers"], d["gamma_keys"], d["gamma"], d["h"], d["beta_h"], d["neg_keys"], d["neg"])
    assert open(out, "rb").read() == blob
    m = srsfile.G2Points(d["neg_keys"], d["neg"])
    assert len(m) == 4 and 3 in m and 4 not in m and m[2] == d["neg"][2].tobytes() and list(m) == [0, 1, 2, 3]


def test_read_ark_rejects_bad_framing_without_allocating(tmp_path):
    from marlin_b200 import srsfile
    path, blob, _ = small_file(tmp_path)

    def rejects(data, what):
        with open(path, "wb") as f:
            f.write(data)
        with pytest.raises(ValueError, match=what):
            srsfile.read_ark(path, 0, True)

    rejects(blob[:-1], "left|truncated")                                 # truncated in the last point
    rejects(blob[:4], "truncated")                                       # truncated in a length field
    rejects(b"", "truncated")
    rejects(blob + b"\0", "trailing")
    rejects(struct.pack("<Q", 1 << 62) + blob[8:], "claims")             # oversized: no 2^62-point array is ever made
    rejects(struct.pack("<Q", (1 << 64) - 1) + blob[8:], "claims")
    g1 = 48
    gam_at = 8 + 4 * g1
    swapped = bytearray(blob)
    k0, k1 = gam_at + 8, gam_at + 8 + (8 + g1)
    swapped[k0:k0 + 8], swapped[k1:k1 + 8] = blob[k1:k1 + 8], blob[k0:k0 + 8]
    rejects(bytes(swapped), "ascending")                                 # keys 1, 0, 2, ...
    dup = bytearray(blob)
    dup[k1:k1 + 8] = blob[k0:k0 + 8]
    rejects(bytes(dup), "ascending")                                     # keys 0, 0, 2, ...
