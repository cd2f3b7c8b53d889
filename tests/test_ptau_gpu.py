"""GPU: snarkjs Powers-of-Tau files as MarlinKZG10 SRSs (Marlin.load_ptau) and the power-chain check (b2m_srs_check_powers).

- A small ceremony file written by the oracle (tests/ptau_writer.py) loads to exactly the SRS `universal_setup(beta = tau,
  gamma = alpha)` makes, proves the same bytes, verifies, and round-trips through an arkworks file.
- Corrupted points are named: a valid subgroup point in the wrong place by the power check (and the same file loads with
  check=False), invalid or infinite points by the decoders; unread sections do not matter; SonicKZG10 is refused; the
  check over an arkworks file names powers_of_g, powers_of_gamma_g and neg_powers_of_h.
- At the size users run: a power-22 file (tauG1 prefix written on the GPU, the rest holes) proves bench.py's 2^20
  DummyCircuit to its pinned hash on both curves."""
import ctypes
import hashlib
import json
import os

import numpy as np
import pytest

from marlin_b200 import _lib, api, fields, r1cs as gr1cs, srsfile
from oracle import ec
from oracle import rng as orng
from oracle.params import BLS12_381, BN254

import ark_srs_oracle as ao
import ptau_writer as pw

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
TAU, ALPHA, BETA = 0x5eed5eed5eed5eed5eed5eed, 7, 0xbe7a
CURVES = [BLS12_381, BN254]


@pytest.fixture(scope="module")
def gctx(b2m_ctx):
    c = api.Context.__new__(api.Context)
    c.handle = b2m_ctx
    return c


def rng():
    return api.ZkRng(bytes([9]) * 32, 20)


def small_instance(curve):
    f = curve.fr
    r = orng.test_rng()
    a, b = orng.field_rand(f, r), orng.field_rand(f, r)
    n = 16
    return gr1cs.dummy_circuit(fields.CURVE_IDS[curve.name], a, b, 10, n), api.max_degree(n, n, 3 * n)


@pytest.fixture(scope="module", params=CURVES, ids=lambda c: c.name)
def ceremony(request, tmp_path_factory):
    """(curve, power, path, sections) of a small ceremony file covering the small instance"""
    from marlin_b200 import ptau
    curve = request.param
    _, md = small_instance(curve)
    power = ptau.power_for_degree(md)
    secs = pw.sections(curve, power, TAU, ALPHA, BETA)
    path = pw.write(str(tmp_path_factory.mktemp("ptau") / "c.ptau"), secs)
    return curve, power, path, secs


def test_ceremony_file_is_the_trapdoor_srs_and_proves_the_same_bytes(gctx, tmp_path, ceremony):
    curve, power, path, _ = ceremony
    circ, md = small_instance(curve)
    m = api.Marlin(curve.name, "marlin_kzg10", ctx=gctx)
    srs = m.load_ptau(path, max_degree=md, rng=rng())
    ref = m.srs_from_trapdoor(md, beta=TAU, gamma=ALPHA)
    handles = [srs, ref]
    try:
        assert np.array_equal(srs.powers_limbs, ref.powers_limbs)
        assert np.array_equal(srs.gamma_limbs, api.srs_gamma_powers(ref, [0, 1, 2]))
        h, beta_h, _ = srsfile.g2_setup(m.curve_id, curve.fr.p, TAU, md, ())
        assert srs.g2[:2] == (h, beta_h)
        pk, pk_ref = m.index(srs, circ), m.index(ref, circ)
        handles += [pk, pk_ref]
        proof = m.prove(pk, circ, api.ZkRng.test_rng())
        assert proof == m.prove(pk_ref, circ, api.ZkRng.test_rng())
        vk = m.verifier_key(pk, srs)
        handles.append(vk)
        assert m.verify(vk, circ.public_input(), proof, rng())
        # the whole file (max degree 2^(power+1) - 2) loads and checks too
        full = m.load_ptau(path, rng=rng())
        handles.append(full)
        assert full.max_degree == 2 ** (power + 1) - 2
        # arkworks users get the ceremony SRS as a `UniversalParams` file
        ark = os.path.join(tmp_path, "srs.ark")
        srs.save_ark(ark, compressed=True)
        again = m.load_ark_srs(ark, compressed=True, check_powers=True, rng=rng())
        handles.append(again)
        pk2 = m.index(again, circ)
        handles.append(pk2)
        assert m.prove(pk2, circ, api.ZkRng.test_rng()) == proof
    finally:
        for x in handles[::-1]:
            x.close()


def load_error(m, curve, secs, tmp_path, md, **kw):
    path = pw.write(os.path.join(tmp_path, "bad.ptau"), secs)
    with pytest.raises(_lib.B2MError) as e:
        m.load_ptau(path, max_degree=md, rng=rng(), **kw)
    assert e.value.code == _lib.ERR_SERIALIZATION
    return str(e.value)


def copy(secs):
    return [[s, bytearray(d)] for s, d in secs]


def test_corrupted_points_are_named(gctx, tmp_path, ceremony):
    curve, power, path, secs = ceremony
    m = api.Marlin(curve.name, "marlin_kzg10", ctx=gctx)
    D = 2 ** (power + 1) - 2
    g2 = ao.G2(curve)
    r = curve.fr.p
    tau_pt = lambda i: ec.scalar_mul(curve, pow(TAU, i, r), curve.g)  # noqa: E731
    # a valid subgroup point in the wrong place: only the power check sees it
    for k in (1, D // 2 + 1, D):
        bad = copy(secs)
        pw.set_point(bad, 2, k, pw.g1_lem(curve, ec.scalar_mul(curve, 2, tau_pt(k))))
        msg = load_error(m, curve, bad, tmp_path, D)
        assert f"tauG1[{k}] is not tau times tauG1[{k - 1}]" in msg
        if k == 1:
            assert "tauG2[1]" in msg
        m.load_ptau(pw.write(os.path.join(tmp_path, "unchecked.ptau"), bad), max_degree=D, check=False).close()
    bad = copy(secs)
    pw.set_point(bad, 3, 1, pw.g2_lem(curve, g2.smul(TAU + 1, g2.gen)))
    assert "tauG2[1]" in load_error(m, curve, bad, tmp_path, D)
    bad = copy(secs)
    pw.set_point(bad, 4, 2, pw.g1_lem(curve, ec.scalar_mul(curve, ALPHA + 1, tau_pt(2))))
    assert "alphaTauG1[2] is not tau times alphaTauG1[1]" in load_error(m, curve, bad, tmp_path, D)
    # invalid points: the decoders name field and index
    nb, p = curve.fq.nbytes, curve.fq.p
    good = pw.g1_lem(curve, tau_pt(5))
    bad = copy(secs)
    pw.set_point(bad, 2, 5, p.to_bytes(nb, "little") + good[nb:])
    assert "tauG1[5]: x is not below the field modulus" in load_error(m, curve, bad, tmp_path, D)
    bad = copy(secs)
    pw.set_point(bad, 2, 6, good[:nb] + pw.fq_lem(curve, tau_pt(6)[1] + 1))
    assert "tauG1[6]: not on the curve" in load_error(m, curve, bad, tmp_path, D)
    if curve is BLS12_381:
        fq = curve.fq
        x = next(x for x in range(1, 1000) if pow((x ** 3 + curve.b) % fq.p, (fq.p - 1) // 2, fq.p) == 1)
        bad = copy(secs)
        pw.set_point(bad, 2, 3, pw.g1_lem(curve, (x, pow((x ** 3 + curve.b) % fq.p, (fq.p + 1) // 4, fq.p))))
        assert "tauG1[3]: not in the prime-order subgroup" in load_error(m, curve, bad, tmp_path, D)
    bad = copy(secs)
    pw.set_point(bad, 2, 4, pw.g1_lem(curve, None))
    assert "tauG1[4]: the point at infinity" in load_error(m, curve, bad, tmp_path, D)
    bad = copy(secs)
    pw.set_point(bad, 3, 0, pw.g2_lem(curve, None))
    assert "tauG2[0]: the point at infinity" in load_error(m, curve, bad, tmp_path, D)
    # garbage where nothing is read
    bad = copy(secs)
    for sid in (5, 6, 7):
        d = next(x for s, x in bad if s == sid)
        d[:] = b"\xa5" * len(d)
    m.load_ptau(pw.write(os.path.join(tmp_path, "garbage.ptau"), bad), max_degree=D, rng=rng()).close()
    with pytest.raises(ValueError, match="SonicKZG10"):
        api.Marlin(curve.name, "sonic_kzg10", ctx=gctx).load_ptau(path)


def test_power_check_draws_a_callback_rng_like_a_chacha_stream(gctx, ceremony):
    """the device-sampled ChaCha randomisers and host-drawn callback ones are the same words: a callback replaying the stream
    gives the same verdicts, draws what the ChaCha position advanced by, and errors come before any draw"""
    curve, power, path, secs = ceremony
    m = api.Marlin(curve.name, "marlin_kzg10", ctx=gctx)
    z = rng()
    m.load_ptau(path, rng=z).close()
    words = z.word_pos
    assert words == 4 * (2 ** (power + 1) - 2 + 2)  # two u64 per relation: D of family 0, two of family 1
    draws = []
    m.load_ptau(path, rng=api.CallbackRng(lambda: draws.append(1) or 12345)).close()
    assert 2 * len(draws) == words
    srs = m.load_ptau(path, check=False)
    try:
        h, beta_h, _ = srs.g2
        ok = ctypes.c_int(0)
        hb = np.frombuffer(h, dtype=np.uint8).copy()
        assert _lib.lib().b2m_srs_check_powers(srs.handle, _lib.ptr(hb), _lib.ptr(hb), 0, None, None, None, ctypes.byref(ok), None,
                                               None) == 7  # B2M_ERR_MISSING_RNG
    finally:
        srs.close()


def test_load_ark_srs_power_check_names_the_bad_point(gctx, tmp_path):
    curve, D = BLS12_381, 12
    blob, pts = ao.kzg10_setup(curve, D, 0x5eed + D, 11, True, False)
    nb = curve.fq.nbytes
    g1b, g2b = 2 * nb, 4 * nb
    off_powers = 8
    off_gamma = off_powers + (D + 1) * g1b + 8  # then (u64 key, point) per gamma entry
    off_neg = off_gamma + (D + 2) * (8 + g1b) + 2 * g2b + 8
    g2 = ao.G2(curve)
    m = api.Marlin(curve.name, "sonic_kzg10", ctx=gctx)

    def err(at, data):
        b = bytearray(blob)
        b[at:at + len(data)] = data
        path = os.path.join(tmp_path, "bad.ark")
        with open(path, "wb") as f:
            f.write(b)
        with pytest.raises(_lib.B2MError) as e:
            m.load_ark_srs(path, compressed=False, check_powers=True, rng=rng())
        return str(e.value)

    ok = os.path.join(tmp_path, "ok.ark")
    with open(ok, "wb") as f:
        f.write(blob)
    m.load_ark_srs(ok, compressed=False, check_powers=True, rng=rng()).close()
    assert "powers_of_g[7] is not beta times powers_of_g[6]" in err(off_powers + 7 * g1b, ao.g1_uncompressed(curve, ec.scalar_mul(curve, 2, pts["powers"][7])))
    assert "powers_of_gamma_g[2]" in err(off_gamma + 2 * (8 + g1b) + 8, ao.g1_uncompressed(curve, ec.scalar_mul(curve, 3, pts["gamma"][2])))
    assert "neg_powers_of_h[5]" in err(off_neg + 5 * (8 + g2b) + 8, g2.uncompressed(g2.smul(2, pts["neg"][5])))


# ---- at the size users run ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("curve_name", ["bls12_381", "bn254"])
def test_power_22_ceremony_file_proves_the_pinned_bench_proof(gctx, tmp_path, curve_name):
    n = 1 << 20
    D = (1 << 22) - 1
    path = os.path.join(tmp_path, "p22.ptau")
    pw.write_gpu_prefix(gctx, fields.CURVE_IDS[curve_name], path, 22, D, TAU, ALPHA)
    m = api.Marlin(curve_name, "marlin_kzg10", ctx=gctx)
    cid = m.curve_id
    a, b = 0x1234567890abcdef1234567890abcdef, 0xfedcba0987654321fedcba0987654321
    circ = gr1cs.dummy_circuit(cid, a, b, 10, n)
    srs = m.load_ptau(path, max_degree=D, check=True, rng=rng())
    handles = [srs]
    try:
        assert srs.max_degree == api.max_degree(n, n, 3 * n) == D
        pk = m.index(srs, circ)
        handles.append(pk)
        proof = m.prove(pk, circ, api.ZkRng.test_rng())
        with open(os.path.join(HERE, "golden", "bench_proof_hashes.json")) as fh:
            pinned = json.load(fh)[f"{curve_name}/marlin_kzg10/20"]
        assert hashlib.sha256(proof).hexdigest() == pinned
        vk = m.verifier_key(pk, srs)
        handles.append(vk)
        assert m.verify(vk, circ.public_input(), proof, rng())
    finally:
        for x in handles[::-1]:
            x.close()
        os.remove(path)
