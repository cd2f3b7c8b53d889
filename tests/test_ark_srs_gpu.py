"""GPU: arkworks `UniversalParams` files (Marlin.load_ark_srs / UniversalSRS.save_ark): a full-shape `KZG10::setup` file
written by the Python model loads to exactly its points and saves back byte for byte, in both forms, for both curves and
both PC schemes; an SRS saved and re-loaded indexes, proves and verifies exactly like the original; at 2^20 powers an
invalid point is reported by field and lowest index across the decoder's chunk boundaries."""
import os

import numpy as np
import pytest

from marlin_b200 import _lib, api, r1cs as gr1cs, srsfile
from oracle import ec
from oracle import rng as orng
from oracle import transcript as T
from oracle.params import BLS12_381, BN254

import ark_srs_oracle as ao

pytestmark = pytest.mark.gpu
CHUNK = 1 << 18  # ARK_DECODE_CHUNK (csrc/ark_points.cuh)


@pytest.fixture(scope="module")
def gctx(b2m_ctx):
    c = api.Context.__new__(api.Context)
    c.handle = b2m_ctx
    return c


def limbs_to_points(curve, limbs):
    fq = curve.fq
    out = []
    for x, y in zip(_lib.limbs_to_ints(limbs[:, :limbs.shape[1] // 2]), _lib.limbs_to_ints(limbs[:, limbs.shape[1] // 2:])):
        out.append(None if x == 0 and y == 0 else (fq.from_mont(x), fq.from_mont(y)))
    return out


@pytest.mark.parametrize("compressed", [True, False], ids=["compressed", "uncompressed"])
@pytest.mark.parametrize("pc", ["marlin_kzg10", "sonic_kzg10"])
@pytest.mark.parametrize("curve", [BLS12_381, BN254], ids=lambda c: c.name)
def test_oracle_file_loads_exactly_and_saves_back(gctx, tmp_path, curve, pc, compressed):
    D = 12
    blob, pts = ao.kzg10_setup(curve, D, 0x5eed + D, 11, pc == "sonic_kzg10", compressed)
    path = os.path.join(tmp_path, "srs.bin")
    with open(path, "wb") as f:
        f.write(blob)
    m = api.Marlin(curve.name, pc, ctx=gctx)
    srs = m.load_ark_srs(path, compressed=compressed, degree_bounds=[4])
    try:
        g2 = ao.G2(curve)
        assert limbs_to_points(curve, srs.powers_limbs) == pts["powers"]
        assert srs.gamma_indices == [0, 1, 2, 8, 9, 10]  # {0, 1, 2} and D - 4 + {0, 1, 2} on the device
        assert limbs_to_points(curve, srs.ark["gamma_limbs"]) == [pts["gamma"][k] for k in range(D + 2)]
        h, beta_h, neg = srs.g2
        assert (h, beta_h) == (g2.uncompressed(pts["h"]), g2.uncompressed(pts["beta_h"]))
        assert sorted(neg) == sorted(pts["neg"]) and all(neg[k] == g2.uncompressed(P) for k, P in pts["neg"].items())
        again = os.path.join(tmp_path, "again.bin")
        srs.save_ark(again, compressed=compressed)
        assert open(again, "rb").read() == blob
        # the other form, and back
        other = os.path.join(tmp_path, "other.bin")
        srs.save_ark(other, compressed=not compressed)
        srs2 = m.load_ark_srs(other, compressed=not compressed)
        back = os.path.join(tmp_path, "back.bin")
        srs2.save_ark(back, compressed=compressed)
        srs2.close()
        assert open(back, "rb").read() == blob
    finally:
        srs.close()


@pytest.mark.parametrize("pc", ["marlin_kzg10", "sonic_kzg10"])
@pytest.mark.parametrize("curve", [BLS12_381, BN254], ids=lambda c: c.name)
def test_saved_and_reloaded_srs_proves_and_verifies_like_the_original(gctx, tmp_path, curve, pc):
    f = curve.fr
    r = orng.test_rng()
    a, b = orng.field_rand(f, r), orng.field_rand(f, r)
    n = 64
    m = api.Marlin(curve.name, pc, ctx=gctx)
    circ = gr1cs.dummy_circuit(m.curve_id, a, b, 10, n)
    md = api.max_degree(n, n, 3 * n)
    bounds = [(1 << k) - 2 for k in range(2, md.bit_length() + 1) if (1 << k) - 2 <= md]
    srs = m.srs_from_trapdoor(md, beta=0x1234567, gamma=7, degree_bounds=bounds)
    path = os.path.join(tmp_path, "srs.bin")
    srs.save_ark(path, compressed=True, degree_bounds=bounds)
    loaded = m.load_ark_srs(path, compressed=True, degree_bounds=bounds)
    handles = []
    try:
        assert np.array_equal(loaded.powers_limbs, srs.powers_limbs)
        pk0, pk1 = m.index(srs, circ), m.index(loaded, circ)
        handles += [pk0, pk1]
        assert pk1.vk_bytes == pk0.vk_bytes
        p0 = m.prove(pk0, circ, api.ZkRng.test_rng())
        p1 = m.prove(pk1, circ, api.ZkRng.test_rng())
        assert p1 == p0
        vk = m.verifier_key(pk1, loaded)
        handles.append(vk)
        assert m.verify_batch(vk, [circ.public_input()] * 2, [p0, p1], api.ZkRng(bytes([3]) * 32, 20)) == [True, True]
    finally:
        for h in handles:
            h.close()
        loaded.close()
        srs.close()


def test_2p20_powers_load_and_bad_points_are_reported_by_lowest_index(gctx, tmp_path, monkeypatch):
    curve = BLS12_381
    n = 1 << 20
    m = api.Marlin("bls12_381", "marlin_kzg10", ctx=gctx)
    srs = m.srs_from_trapdoor(n - 1, beta=0xabcdef12345, gamma=7)
    path = os.path.join(tmp_path, "srs.bin")
    srs.save_ark(path, compressed=True)
    loaded = m.load_ark_srs(path, compressed=True)
    try:
        assert np.array_equal(loaded.powers_limbs, srs.powers_limbs)
    finally:
        loaded.close()
        srs.close()
    blob = bytearray(open(path, "rb").read())
    nb = curve.fq.nbytes
    x = next(x for x in range(1, 1000) if pow((x ** 3 + curve.b) % curve.fq.p, (curve.fq.p - 1) // 2, curve.fq.p) == 1)
    outside = T.g1_compressed(curve, (x, pow((x ** 3 + curve.b) % curve.fq.p, (curve.fq.p + 1) // 4, curve.fq.p)))
    x_big = curve.fq.p.to_bytes(nb, "little")
    created = []
    real = api.Marlin.srs_from_points
    monkeypatch.setattr(api.Marlin, "srs_from_points", lambda self, *a, **k: created.append(1) or real(self, *a, **k))

    def load_with(plants):
        data = bytearray(blob)
        for i, pt in plants:
            data[8 + i * nb:8 + (i + 1) * nb] = pt
        bad = os.path.join(tmp_path, "bad.bin")
        with open(bad, "wb") as f:
            f.write(data)
        with pytest.raises(_lib.B2MError) as e:
            m.load_ark_srs(bad, compressed=True)
        assert e.value.code == _lib.ERR_SERIALIZATION
        return str(e.value)

    assert "powers_of_g[%d]: not in the prime-order subgroup" % (CHUNK - 1) in load_with([(CHUNK - 1, outside)])
    assert "powers_of_g[%d]: x is not below the field modulus" % CHUNK in load_with([(CHUNK, x_big)])
    assert "powers_of_g[%d]: not in the prime-order subgroup" % (n - 3) in load_with([(n - 3, outside)])
    assert "powers_of_g[%d]:" % (2 * CHUNK + 5) in load_with([(3 * CHUNK + 1, x_big), (2 * CHUNK + 5, outside)])
    assert "powers_of_g[%d]:" % (CHUNK + 7) in load_with([(CHUNK + 9, x_big), (CHUNK + 7, outside)])  # two in one chunk
    assert created == []  # no device key was made for a file that failed
    # a bad G2 point names its field and key
    d = srsfile.read_ark(path, 0, True)
    g2_at = len(blob) - 8 - 2 * (2 * nb)  # h, beta_h, then the empty neg_powers_of_h map
    data = bytearray(blob)
    data[g2_at + 2 * nb:g2_at + 4 * nb] = bytes(2 * nb - 1) + b"\x80"
    bad = os.path.join(tmp_path, "bad_g2.bin")
    with open(bad, "wb") as f:
        f.write(data)
    with pytest.raises(_lib.B2MError, match="beta_h: "):
        m.load_ark_srs(bad, compressed=True)
    assert len(d["neg_keys"]) == 0
