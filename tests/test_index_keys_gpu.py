"""GPU: arkworks index key files (IndexProverKey.save / save_verifier_key, Marlin.load_index / load_verifier_key).

- the product writes exactly the bytes of the independent oracle writer (tests/index_key_oracle.py) for both curves, both
  PC schemes and both point forms, on DummyCircuit and on general R1CS with |K| below and far above |H|;
- an empty coefficient vector (the zero polynomial of an empty C matrix) is written empty and zero-padded back on load;
- an index loaded from the oracle's file proves byte-identical proofs to a fresh `Marlin.index` and to the oracle, and a
  verifier key loaded from its file alone gives the same verdicts as `Marlin.verifier_key(pk, srs)`;
- corruptions are rejected naming the field and the lowest bad index: an Fr >= r past a 2^18-element decode chunk, points
  off the curve or outside the subgroup in the committer key, coefficients inconsistent with their evaluations, a committer
  key from another SRS, and a tampered commitment (only with check_commitments=True);
- at 2^20 constraints, save -> load_index -> prove reproduces the pinned bench proof."""
import hashlib
import json
import os

import numpy as np
import pytest

import index_key_oracle as iko
import r1cs_random as R
from marlin_b200 import _lib, api, keyfile, r1cs as gr1cs
from oracle import ahp, kzg
from oracle import marlin as omarlin
from oracle import r1cs as or1cs
from oracle import rng as orng
from oracle import transcript as T
from oracle.params import BLS12_381, BN254

pytestmark = pytest.mark.gpu
CHUNK = 1 << 18  # ARK_DECODE_CHUNK (csrc/ark_points.cuh)
SCHEMES = {"marlin_kzg10": kzg.MARLIN, "sonic_kzg10": kzg.SONIC}
CURVES = {0: BLS12_381, 1: BN254}
BETA, GAMMA = 0x1234567, 7


@pytest.fixture(scope="module")
def gctx(b2m_ctx):
    c = api.Context.__new__(api.Context)
    c.handle = b2m_ctx
    return c


def file_offset(view):
    """byte offset of a keyfile view inside its memory-mapped file"""
    base = view
    while isinstance(base.base, np.ndarray):
        base = base.base
    return view.__array_interface__["data"][0] - base.__array_interface__["data"][0]


def dummy(curve, n):
    f = curve.fr
    r = orng.test_rng()
    a, b = orng.field_rand(f, r), orng.field_rand(f, r)
    return or1cs.dummy_circuit(f, a, b, 10, n), gr1cs.dummy_circuit(0 if curve is BLS12_381 else 1, a, b, 10, n), [a * b % f.p]


def run_parity(gctx, tmp_path, curve, pc, compressed, ocirc, gcirc, pub, oracle_proof=True):
    f = curve.fr
    cs = or1cs.synthesize(f, ocirc)
    nnz = sum(len(r) for r in ahp.sum_matrices(*cs.to_matrices()))
    osrs = omarlin.universal_setup(curve, cs.num_constraints, len(cs.instance) + len(cs.witness), nnz, beta=BETA, g_scalar=1, gamma=GAMMA)
    eng = kzg.Engine(use_trapdoor=True)
    opk = omarlin.index(osrs, ocirc, SCHEMES[pc], eng)
    w = iko.KeyWriter(osrs, opk, compressed)
    want_pk, want_vk = w.prover_key(), w.verifier_key()
    m = api.Marlin(curve.name, pc, ctx=gctx)
    srs = m.srs_from_trapdoor(osrs.max_degree, beta=BETA, gamma=GAMMA, degree_bounds=opk.ck.enforced_degree_bounds)
    handles = []
    try:
        pk = m.index(srs, gcirc)
        handles.append(pk)
        pk_path, vk_path = str(tmp_path / "pk.bin"), str(tmp_path / "vk.bin")
        pk.save(pk_path, compressed=compressed)
        pk.save_verifier_key(vk_path, compressed=compressed)
        assert open(vk_path, "rb").read() == want_vk, "IndexVerifierKey bytes differ from the oracle writer"
        assert open(pk_path, "rb").read() == want_pk, "IndexProverKey bytes differ from the oracle writer"
        # load the oracle's own files
        with open(pk_path, "wb") as fh:
            fh.write(want_pk)
        with open(vk_path, "wb") as fh:
            fh.write(want_vk)
        pk2 = m.load_index(srs, pk_path, compressed=compressed, check_commitments=True)
        handles.append(pk2)
        assert pk2.vk_bytes == pk.vk_bytes
        again = str(tmp_path / "again.bin")
        pk2.save(again, compressed=compressed)
        assert open(again, "rb").read() == want_pk, "a loaded key does not save back to its file"
        p1 = m.prove(pk, gcirc, api.ZkRng.test_rng())
        p2 = m.prove(pk2, gcirc, api.ZkRng.test_rng())
        assert p2 == p1, "a loaded index proves differently from a fresh one"
        if oracle_proof:
            assert p2 == omarlin.serialize_proof(curve, SCHEMES[pc], omarlin.prove(opk, ocirc, orng.test_rng(), eng))
        vk_file = m.load_verifier_key(vk_path, compressed=compressed)
        vk_live = m.verifier_key(pk, srs)
        handles += [vk_file, vk_live]
        ins = [pub, [(pub[0] + 1) % f.p] + list(pub[1:])] if pub else [pub]
        proofs = [p2] * len(ins)
        got = m.verify_batch(vk_file, ins, proofs, api.ZkRng(bytes([5]) * 32, 20))
        assert got == [True] + [False] * (len(ins) - 1)
        assert got == m.verify_batch(vk_live, ins, proofs, api.ZkRng(bytes([5]) * 32, 20))
    finally:
        for h in reversed(handles):
            h.close()
        srs.close()


@pytest.mark.parametrize("compressed", [True, False], ids=["compressed", "uncompressed"])
@pytest.mark.parametrize("pc", list(SCHEMES))
@pytest.mark.parametrize("curve", [BLS12_381, BN254], ids=lambda c: c.name)
@pytest.mark.parametrize("n", [16, 1024])
def test_dummy_circuit_keys_match_oracle(gctx, tmp_path, n, curve, pc, compressed):
    ocirc, gcirc, pub = dummy(curve, n)
    run_parity(gctx, tmp_path, curve, pc, compressed, ocirc, gcirc, pub, oracle_proof=n <= 16)


@pytest.mark.parametrize("name", ["x4-squat-k-below-h", "k-far-above-h", "x2-tall-hot", "x1-square"])
def test_general_r1cs_keys_match_oracle(gctx, tmp_path, name):
    g = R.small_case(name)
    curve = CURVES[g.curve_id]
    pc = R.SMALL_CASES[name]["scheme"]
    for compressed in (True, False):
        run_parity(gctx, tmp_path, curve, pc, compressed, g.circuit(curve.fr), g.r1cs, g.public_input)


@pytest.mark.parametrize("pc", list(SCHEMES))
@pytest.mark.parametrize("curve", [BLS12_381, BN254], ids=lambda c: c.name)
def test_zero_polynomial_keys_match_oracle(gctx, tmp_path, curve, pc):
    """An empty C matrix: c_val is the zero polynomial, stored with no coefficients.  save strips the |K| zero coefficients the
    index holds, load_index zero-pads the empty vector back to |K| (its NTT check then compares zeros with the zero
    evaluations), the loaded key saves back to the same bytes and proves the same proofs."""
    f = curve.fr
    a = 0x1234
    ocirc = iko.zero_c_circuit(f, a, 16)
    cs = or1cs.synthesize(f, ocirc)
    gcirc = gr1cs.from_rows(0 if curve is BLS12_381 else 1, *cs.to_matrices(), cs.instance, cs.witness)
    for compressed in (True, False):
        run_parity(gctx, tmp_path, curve, pc, compressed, ocirc, gcirc, [a])


# ---- corruptions ------------------------------------------------------------------------------------------------------
def _fresh_files(gctx, tmp_path, curve, pc, n=64):
    m = api.Marlin(curve.name, pc, ctx=gctx)
    _, gcirc, _ = dummy(curve, n)
    bounds = (n - 2, 4 * n - 2)
    srs = m.universal_setup(n, n, 3 * n, beta=BETA, gamma=GAMMA, degree_bounds=bounds)
    pk = m.index(srs, gcirc)
    path = str(tmp_path / "pk.bin")
    pk.save(path, compressed=True)
    pk.close()
    return m, srs, path


def _load_bad(m, srs, tmp_path, data, exc=_lib.B2MError, **kw):
    bad = str(tmp_path / "bad.bin")
    with open(bad, "wb") as fh:
        fh.write(bytes(data))
    with pytest.raises(exc) as e:
        m.load_index(srs, bad, compressed=True, **kw).close()
    return str(e.value)


def test_bad_points_in_the_committer_key_are_named(gctx, tmp_path):
    curve = BLS12_381
    m, srs, path = _fresh_files(gctx, tmp_path, curve, "marlin_kzg10")
    try:
        d = keyfile.read_prover_key(path, 0, _lib.PC_MARLIN_KZG10, True)
        blob = open(path, "rb").read()
        nb, p = curve.fq.nbytes, curve.fq.p
        x_off = next(x for x in range(1, 1000) if pow((x ** 3 + curve.b) % p, (p - 1) // 2, p) != 1)  # no square root
        x_in = next(x for x in range(1, 1000) if pow((x ** 3 + curve.b) % p, (p - 1) // 2, p) == 1)
        off_curve = x_off.to_bytes(nb, "little")
        outside = T.g1_compressed(curve, (x_in, pow((x_in ** 3 + curve.b) % p, (p + 1) // 4, p)))
        for field, view, i, pt, reason in (("committer_key.powers", d["ck"]["powers"], 5, off_curve, "not on the curve"),
                                           ("committer_key.shifted_powers", d["ck"]["shifted"], 12, outside, "not in the prime-order subgroup"),
                                           ("committer_key.powers_of_gamma_g", d["ck"]["gamma"], 2, outside, "not in the prime-order subgroup")):
            at = file_offset(view) + i * nb
            data = bytearray(blob)
            data[at:at + nb] = pt
            assert f"{field}[{i}]: {reason}" in _load_bad(m, srs, tmp_path, data)
    finally:
        srs.close()


def test_inconsistent_coefficients_other_srs_and_tampered_commitment(gctx, tmp_path):
    curve = BLS12_381
    m, srs, path = _fresh_files(gctx, tmp_path, curve, "marlin_kzg10")
    try:
        d = keyfile.read_prover_key(path, 0, _lib.PC_MARLIN_KZG10, True)
        blob = open(path, "rb").read()
        # one coefficient of b_val changed (still below r): its evaluations no longer match
        at = file_offset(d["index"]["coeffs"][3]) + 2 * 32
        data = bytearray(blob)
        data[at] ^= 1
        assert "index.joint_arith.evals_on_K.val_b[0]: not the FFT over K of index.joint_arith.b_val.polynomial" in _load_bad(m, srs, tmp_path, data)
        # a committer key made from another SRS
        other = m.universal_setup(64, 64, 192, beta=BETA + 1, gamma=GAMMA, degree_bounds=(62, 254))
        try:
            msg = _load_bad(m, other, tmp_path, blob, ValueError)
            assert "committer_key.powers[1]: differs from the SRS" in msg
        finally:
            other.close()
        # a tampered commitment (another valid point): accepted unless the commitments are recomputed
        g1 = curve.fq.nbytes
        c2, c3 = 32 + 8 + 2 * (g1 + 1), 32 + 8 + 3 * (g1 + 1)
        data = bytearray(blob)
        data[c2:c2 + g1] = blob[c3:c3 + g1]
        tampered = str(tmp_path / "tampered.bin")
        with open(tampered, "wb") as fh:
            fh.write(data)
        m.load_index(srs, tampered, compressed=True).close()
        assert "index_vk.index_comms[2]: not the commitment to index.joint_arith.a_val" in _load_bad(m, srs, tmp_path, data, check_commitments=True)
    finally:
        srs.close()


def test_fr_not_below_r_is_reported_past_a_chunk_boundary(gctx, tmp_path):
    """|K| = 2^19: an element >= r in evals_on_K.val_b just past the first 2^18-element decode chunk, with a second one
    later, is reported at the lower index."""
    g = R.generate(0, seed=31, num_public=15, live=1 << 12, free=(1 << 13) - 16 - (1 << 12), terms=(32, 32, 8))
    assert g.K == 1 << 19, g.K
    circ = g.r1cs
    m = api.Marlin("bls12_381", "marlin_kzg10", ctx=gctx)
    srs = m.universal_setup(circ.num_constraints, circ.num_variables, g.nnz, beta=BETA, gamma=GAMMA, degree_bounds=(g.H - 2, g.K - 2))
    try:
        pk = m.index(srs, circ)
        path = str(tmp_path / "pk.bin")
        pk.save(path, compressed=True)
        want = m.prove(pk, circ, api.ZkRng.test_rng())
        pk.close()
        pk2 = m.load_index(srs, path)
        assert m.prove(pk2, circ, api.ZkRng.test_rng()) == want
        pk2.close()
        d = keyfile.read_prover_key(path, 0, _lib.PC_MARLIN_KZG10, True)
        blob = open(path, "rb").read()
        curve_r = BLS12_381.fr.p
        ev = file_offset(d["index"]["evals"][3])
        data = bytearray(blob)
        for i, v in ((CHUNK + 1, curve_r), (CHUNK + 70000, (1 << 256) - 1)):
            data[ev + 32 * i:ev + 32 * (i + 1)] = v.to_bytes(32, "little")
        assert f"index.joint_arith.evals_on_K.val_b[{CHUNK + 1}]: not below the field modulus" in _load_bad(m, srs, tmp_path, data)
    finally:
        srs.close()


def test_2p20_save_load_prove_reproduces_the_pinned_proof(gctx, tmp_path):
    log_n = 20
    n = 1 << log_n
    a, b = 0x1234567890abcdef1234567890abcdef, 0xfedcba0987654321fedcba0987654321
    m = api.Marlin("bls12_381", "marlin_kzg10", ctx=gctx)
    srs = m.universal_setup(n, n, 3 * n, beta=0x5eed5eed5eed5eed5eed5eed, gamma=7, degree_bounds=(n - 2, 4 * n - 2))
    circ = gr1cs.dummy_circuit(0, a, b, 10, n)
    try:
        pk = m.index(srs, circ)
        path = str(tmp_path / "pk.bin")
        pk.save(path, compressed=True)
        pk.close()
        pk2 = m.load_index(srs, path)
        try:
            proof = m.prove(pk2, circ, api.ZkRng.test_rng())
        finally:
            pk2.close()
        with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bench_proof_hashes.json")) as fh:
            pinned = json.load(fh)[f"bls12_381/marlin_kzg10/{log_n}"]
        assert hashlib.sha256(proof).hexdigest() == pinned
    finally:
        srs.close()
