"""CPU: the committed BLS12-377 replay kit (tests/golden/replay_kit_bls12_377, written on a GPU by
`tools/make_replay_kit.py <dir> 6 bls12_377` and replayed by tools/replay_rs through ark-bls12-377 where a Rust toolchain exists)
against the oracle: the SRS file holds the oracle's G1 powers and gamma powers, the G2 half is the curve's generator times the
trapdoor powers, and the GPU-made index_vk bytes and proofs are the oracle's for the same circuit and rng seed."""
import json
import os

import pytest

import bls12_377_oracle as B
from marlin_b200 import _lib, srsfile
from oracle import ec, kzg, marlin as omarlin, r1cs as or1cs
from oracle import rng as orng

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KIT = os.path.join(ROOT, "tests", "golden", "replay_kit_bls12_377")
curve = B.BLS12_377


@pytest.fixture(scope="module")
def meta():
    return json.load(open(os.path.join(KIT, "meta.json")))


def g2_from_bytes(raw):
    nb = curve.fq.nbytes
    x0, x1, y0, y1 = (int.from_bytes(raw[k * nb:(k + 1) * nb], "little") for k in range(4))
    assert y1 >> (8 * nb - 2) == 0
    return (x0, x1), (y0, y1)


def test_kit_srs_file_is_the_oracles_srs(meta):
    assert meta["curve"] == "bls12_377"
    d = srsfile.read_srs(os.path.join(KIT, "srs.bin"))
    assert d["curve_id"] == _lib.CURVE_BLS12_377
    nb = curve.fq.nbytes
    n = 1 << meta["log_n"]
    beta, gamma = int(meta["beta"]), int(meta["gamma"])
    r = curve.fr.p
    D = len(d["powers"]) // (2 * nb) - 1
    assert D == 4 * n - 1
    want = ec.fixed_base_powers(curve, curve.g, beta, D + 1)
    for i in range(D + 1):
        raw = d["powers"][i * 2 * nb:(i + 1) * 2 * nb]
        assert (int.from_bytes(raw[:nb], "little"), int.from_bytes(raw[nb:], "little")) == want[i]
    gamma_g = ec.scalar_mul(curve, gamma, curve.g)
    for k, raw in d["gamma"].items():
        assert (int.from_bytes(raw[:nb], "little"), int.from_bytes(raw[nb:], "little")) == ec.scalar_mul(curve, pow(beta, k, r), gamma_g)
    # G2 half: h is ark-bls12-377's generator, beta_h = beta h, neg_powers[k] = beta^-k h (Fq2 arithmetic with u^2 = -5)
    h = ((B.G2_GENERATOR[0], B.G2_GENERATOR[1]), (B.G2_GENERATOR[2], B.G2_GENERATOR[3]))
    assert g2_from_bytes(d["h"]) == h
    assert g2_from_bytes(d["beta_h"]) == B.g2_mul(beta, h)
    assert sorted(d["neg_powers"]) == sorted(D - b for b in (n - 2, 4 * n - 2))
    for k, raw in d["neg_powers"].items():
        assert g2_from_bytes(raw) == B.g2_mul(pow(pow(beta, k, r), -1, r), h)


@pytest.mark.parametrize("pc,scheme", [("marlin_kzg10", kzg.MARLIN), ("sonic_kzg10", kzg.SONIC)])
def test_kit_bytes_are_the_oracles(meta, pc, scheme):
    f = curve.fr
    n = 1 << meta["log_n"]
    a, b = int(meta["a"]), int(meta["b"])
    circ = or1cs.dummy_circuit(f, a % f.p, b % f.p, meta["num_variables"], n)
    srs = omarlin.universal_setup(curve, n, n, 3 * n, beta=int(meta["beta"]), g_scalar=1, gamma=int(meta["gamma"]))
    eng = kzg.Engine(use_trapdoor=True)
    pk = omarlin.index(srs, circ, scheme, eng)
    assert pk.vk_bytes == open(os.path.join(KIT, f"{pc}_index_vk_tobytes.bin"), "rb").read()
    zk = orng.ChaChaRng(bytes.fromhex(meta["zk_seed_hex"]), 12)
    proof = omarlin.prove(pk, circ, zk, eng)
    assert omarlin.serialize_proof(curve, scheme, proof) == open(os.path.join(KIT, f"{pc}_proof.bin"), "rb").read()
    assert zk.word_pos == meta["zk_word_pos_after"][pc]
    assert omarlin.verify(pk, [int(v) for v in meta["public_input"]], proof)
    g2 = kzg.G2Key(srs, pk.ck.enforced_degree_bounds)
    assert omarlin.verify(pk, [int(v) for v in meta["public_input"]], proof, g2)

