"""CPU: snarkjs Powers-of-Tau files -- the framing checks of marlin_b200.ptau (each error names its section), and the LEM point
decoders of csrc/g1_decode.cuh / g2_decode.cuh compiled for the host against the Python oracle: valid points, a coordinate
>= p, off the curve, BLS12-381 G1 torsion, G2 outside the subgroup and all-zero infinity."""
import ctypes
import os
import random
import subprocess
import types

import numpy as np
import pytest

from marlin_b200 import _lib, api, ptau
from oracle import ec
from oracle.params import BLS12_381, BN254

import ark_srs_oracle as ao
import ptau_writer as pw

HERE = os.path.dirname(os.path.abspath(__file__))
CURVES = list(enumerate([BLS12_381, BN254]))
IDS = lambda x: getattr(x, "name", x)  # noqa: E731
OK, BAD_FLAGS, X_NC, NOT_ON_CURVE, NOT_IN_SUBGROUP, Y_NC = range(6)


@pytest.fixture(scope="module")
def hostlib(tmp_path_factory):
    src = os.path.join(HERE, "host", "ptau_host_shim.cpp")
    so = str(tmp_path_factory.mktemp("ptau_host") / "libptau_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-DB2M_HOST_LIGHT_INLINE", "-shared", "-fPIC", "-x", "c++", src, "-o", so])
    return ctypes.CDLL(so)


def vp(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def n32(curve):
    return curve.fq.nbytes // 4


def g1_decode(lib, ci, curve, blobs):
    n = len(blobs)
    out = np.zeros(n * 2 * n32(curve), dtype=np.uint32)
    st = np.zeros(n, dtype=np.int32)
    data = np.frombuffer(b"".join(blobs), dtype=np.uint8).copy()
    lib.g1_decode_lem_host(ci, vp(data), n, vp(out), vp(st))
    res = []
    for i in range(n):
        w = out[i * 2 * n32(curve):(i + 1) * 2 * n32(curve)]
        x = sum(int(w[k]) << (32 * k) for k in range(n32(curve)))
        y = sum(int(w[n32(curve) + k]) << (32 * k) for k in range(n32(curve)))
        res.append((int(st[i]), None if x == 0 and y == 0 else (curve.fq.from_mont(x), curve.fq.from_mont(y))))
    return res


def g2_decode(lib, ci, curve, blobs):
    n = len(blobs)
    nb = 4 * curve.fq.nbytes
    out = np.zeros(n * nb, dtype=np.uint8)
    st = np.zeros(n, dtype=np.int32)
    data = np.frombuffer(b"".join(blobs), dtype=np.uint8).copy()
    lib.g2_decode_lem_host(ci, vp(data), n, vp(out), vp(st))
    raw = out.tobytes()
    return [(int(st[i]), raw[i * nb:(i + 1) * nb]) for i in range(n)]


def raw_limbs(curve, v):
    """v as raw little-endian limbs (no Montgomery conversion): lets a test write a limb vector >= p"""
    return v.to_bytes(curve.fq.nbytes, "little")


def raw_g1(curve, start=1):
    fq = curve.fq
    x = next(x for x in range(start, start + 1000) if pow((x ** 3 + curve.b) % fq.p, (fq.p - 1) // 2, fq.p) == 1)
    return (x, pow((x ** 3 + curve.b) % fq.p, (fq.p + 1) // 4, fq.p))


# ---- decoders -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ci,curve", CURVES, ids=IDS)
def test_g1_lem_decoder_matches_the_oracle(hostlib, ci, curve):
    rnd = random.Random(30 + ci)
    pts = [ec.scalar_mul(curve, rnd.randrange(1, curve.fr.p), curve.g) for _ in range(12)] + [curve.g, None]
    assert g1_decode(hostlib, ci, curve, [pw.g1_lem(curve, P) for P in pts]) == [(OK, P) for P in pts]


@pytest.mark.parametrize("ci,curve", CURVES, ids=IDS)
def test_g1_lem_decoder_rejects_every_invalid_class(hostlib, ci, curve):
    G = curve.g
    xm, ym = pw.fq_lem(curve, G[0]), pw.fq_lem(curve, G[1])
    p = curve.fq.p
    cases = [raw_limbs(curve, p) + ym,                       # x limbs = p: not a reduced Montgomery representative
             raw_limbs(curve, p + 5) + ym,
             xm + raw_limbs(curve, p),                       # y >= p
             xm + pw.fq_lem(curve, G[1] + 1),                # off the curve
             bytes(curve.fq.nbytes) + ym]                    # x = 0, y != 0: not infinity, and off the curve
    assert [s for s, _ in g1_decode(hostlib, ci, curve, cases)] == [X_NC, X_NC, Y_NC, NOT_ON_CURVE, NOT_ON_CURVE]
    R = raw_g1(curve)
    assert [s for s, _ in g1_decode(hostlib, ci, curve, [pw.g1_lem(curve, R)])] == ([NOT_IN_SUBGROUP] if ci == 0 else [OK])


@pytest.mark.parametrize("ci,curve", CURVES, ids=IDS)
def test_g2_lem_decoder_matches_the_oracle_and_rejects_every_invalid_class(hostlib, ci, curve):
    g2 = ao.G2(curve)
    rnd = random.Random(40 + ci)
    pts = [g2.smul(rnd.randrange(1, curve.fr.p), g2.gen) for _ in range(3)] + [g2.gen, None]
    assert g2_decode(hostlib, ci, curve, [pw.g2_lem(curve, Q) for Q in pts]) == [(OK, g2.uncompressed(Q)) for Q in pts]
    good = pw.g2_lem(curve, g2.gen)
    nb, p = curve.fq.nbytes, curve.fq.p
    off = bytearray(good)
    off[2 * nb:3 * nb] = pw.fq_lem(curve, g2.gen[1][0] + 1)
    cases = [raw_limbs(curve, p) + good[nb:], good[:nb] + raw_limbs(curve, p) + good[2 * nb:], good[:2 * nb] + raw_limbs(curve, p) + good[3 * nb:],
             good[:3 * nb] + raw_limbs(curve, p + 1), bytes(off)]
    assert [s for s, _ in g2_decode(hostlib, ci, curve, cases)] == [X_NC, X_NC, Y_NC, Y_NC, NOT_ON_CURVE]
    R = g2.raw_point()
    assert [s for s, _ in g2_decode(hostlib, ci, curve, [pw.g2_lem(curve, R)])] == [NOT_IN_SUBGROUP]


# ---- framing --------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def bn_sections():
    return pw.sections(BN254, 2, 0x1234, 5, 9)


def framing_error(tmp_path, secs, **kw):
    path = pw.write(os.path.join(tmp_path, "f.ptau"), secs, **kw)
    with pytest.raises(ValueError) as e:
        ptau.read_ptau(path)
    return str(e.value)


def copy(secs):
    return [[s, bytearray(d)] for s, d in secs]


def test_a_well_formed_file_frames(tmp_path, bn_sections):
    for prepared in (False, True):
        secs = pw.sections(BN254, 2, 0x1234, 5, 9, prepared=prepared) if prepared else copy(bn_sections)
        f = ptau.read_ptau(pw.write(os.path.join(tmp_path, "ok.ptau"), secs[::-1]))  # sections in any order
        assert (f.curve_id, f.n8, f.power, f.ceremony_power, f.max_degree) == (_lib.CURVE_BN254, 32, 2, 2, 6)
        assert f.tau_g1(7).tobytes() == bytes(bn_sections[1][1])
        assert f.tau_g2(1).tobytes() == bytes(bn_sections[2][1][:128])
        assert f.alpha_tau_g1(3).shape == (3, 64)


def test_framing_errors_name_their_section(tmp_path, bn_sections):
    assert "magic" in framing_error(tmp_path, copy(bn_sections), magic=b"ptaU")
    assert "version 2" in framing_error(tmp_path, copy(bn_sections), version=2)
    for sid, name in ((1, "header"), (2, "tauG1"), (3, "tauG2"), (4, "alphaTauG1")):
        assert f"section {sid} ({name}) is missing" in framing_error(tmp_path, [s for s in copy(bn_sections) if s[0] != sid])
        secs = copy(bn_sections)
        secs.append([sid, bytearray(secs[sid - 1][1])])
        assert f"section {sid} ({name}) appears more than once" in framing_error(tmp_path, secs)
    for sid, name in ((2, "tauG1"), (3, "tauG2"), (4, "alphaTauG1")):
        secs = copy(bn_sections)
        secs[sid - 1][1] += bytes(64)  # one point too many for power 2
        assert f"section {sid} ({name}) has" in framing_error(tmp_path, secs)
    secs = copy(bn_sections)
    secs[0][0] = 9  # the header's id changed: the header is missing
    assert "section 1 (header) is missing" in framing_error(tmp_path, secs)


def test_truncation_and_sizes_past_the_end_are_refused(tmp_path, bn_sections):
    path = pw.write(os.path.join(tmp_path, "t.ptau"), copy(bn_sections))
    blob = open(path, "rb").read()
    with open(path, "wb") as f:
        f.write(blob[:-2])  # section 7 (the last) runs past the end
    with pytest.raises(ValueError, match=r"section 7 \(contributions\) of 4 bytes runs past the end"):
        ptau.read_ptau(path)
    assert "section 2 (tauG1) of" in framing_error(tmp_path, copy(bn_sections), sizes={1: 1 << 40})
    with open(path, "wb") as f:
        f.write(blob[:12 + 12 + 44 + 5])  # a section entry header cut short
    with pytest.raises(ValueError, match="runs past the end"):
        ptau.read_ptau(path)


def test_unknown_q_and_bad_header_fields_are_refused(tmp_path, bn_sections):
    secs = copy(bn_sections)
    secs[0][1] = bytearray(pw.header(BN254, 2, q=BN254.fq.p + 2))
    assert "section 1 (header): q = " in framing_error(tmp_path, secs)
    # BLS12-377 is not a snarkjs curve
    q377 = 0x01ae3a4617c510eac63b05c06ca1493b1a22d9f300f5138f1ef3622fba094800170b5d44300000008508c00000000001
    secs[0][1] = bytearray(pw.header(BLS12_381, 2, q=q377))
    assert "neither the BN254 nor the BLS12-381" in framing_error(tmp_path, secs)
    secs[0][1] = bytearray(pw.header(BN254, 2)) + b"\0"
    assert "section 1 (header) has" in framing_error(tmp_path, secs)
    secs[0][1] = bytearray(pw.header(BN254, 3))  # power 3 promises more points than the sections hold
    assert "section 2 (tauG1) has" in framing_error(tmp_path, secs)


def test_degree_beyond_the_file_names_the_power_it_needs(tmp_path, bn_sections):
    assert ptau.power_for_degree(6) == 2 and ptau.power_for_degree(7) == 3
    assert ptau.power_for_degree((1 << 22) - 1) == 22  # a 2^20 DummyCircuit (md = 2^22 - 1) needs a power-22 file
    assert ptau.power_for_degree((1 << 22) - 2) == 21
    path = pw.write(os.path.join(tmp_path, "d.ptau"), copy(bn_sections))
    m = types.SimpleNamespace(pc=_lib.PC_MARLIN_KZG10, curve_id=_lib.CURVE_BN254)  # refused before any device work
    with pytest.raises(ValueError, match="max degree 7 needs a power-3 file; this one is power 2"):
        api.Marlin.load_ptau(m, path, max_degree=7)
    with pytest.raises(ValueError, match="SonicKZG10"):
        api.Marlin.load_ptau(types.SimpleNamespace(pc=_lib.PC_SONIC_KZG10, curve_id=_lib.CURVE_BN254), path)
    with pytest.raises(ValueError, match="bn254 file, this Marlin instance is bls12_381"):
        api.Marlin.load_ptau(types.SimpleNamespace(pc=_lib.PC_MARLIN_KZG10, curve_id=_lib.CURVE_BLS12_381), path)


def test_points_are_views_of_the_file(tmp_path, bn_sections):
    f = ptau.read_ptau(pw.write(os.path.join(tmp_path, "m.ptau"), copy(bn_sections)))
    assert not f.tau_g1(3).flags.owndata
    with pytest.raises(ValueError, match="holds 7 points"):
        f.tau_g1(8)
