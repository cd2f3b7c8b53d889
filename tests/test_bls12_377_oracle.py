"""CPU: the oracle on BLS12-377 (tests/bls12_377_oracle.py) -- the reference's five test.rs circuit shapes prove, verify for the
right public input and are rejected for a wrong one, with both PC schemes, through the trapdoor check and through the pairing
product; their proofs deserialize back to the same bytes; and the golden file regenerates byte for byte."""
import json
import os

import pytest

import bls12_377_oracle as B
from oracle import kzg, marlin as omarlin, r1cs as or1cs
from oracle import rng as orng

CURVE = B.BLS12_377
HERE = os.path.dirname(os.path.abspath(__file__))
REF_SHAPES = {"tall_big": (100, 25), "tall_small": (26, 25), "squat_big": (25, 100), "squat_small": (25, 26), "square": (25, 25)}


@pytest.mark.parametrize("shape", list(REF_SHAPES))
@pytest.mark.parametrize("scheme", [kzg.MARLIN, kzg.SONIC])
def test_reference_shapes_prove_and_verify(shape, scheme):
    f = CURVE.fr
    nc, nv = REF_SHAPES[shape]
    rng = orng.test_rng()
    a, b = orng.field_rand(f, rng), orng.field_rand(f, rng)
    c = a * b % f.p
    d = c * b % f.p
    circ = or1cs.test_circuit(f, a, b, nc, nv)
    cs = or1cs.synthesize(f, circ)
    nnz = sum(len({i for _, i in ra} | {i for _, i in rb} | {i for _, i in rc}) for ra, rb, rc in zip(*cs.to_matrices()))
    srs = omarlin.universal_setup(CURVE, cs.num_constraints, len(cs.instance) + len(cs.witness), nnz, beta=0x1234567, g_scalar=3, gamma=11)
    eng = kzg.Engine(use_trapdoor=True)
    pk = omarlin.index(srs, circ, scheme, eng)
    proof = omarlin.prove(pk, circ, orng.ChaChaRng(bytes(range(32)), 12), eng)
    assert omarlin.verify(pk, [c, d], proof)
    assert not omarlin.verify(pk, [a, a], proof)
    data = omarlin.serialize_proof(CURVE, scheme, proof)
    assert omarlin.serialize_proof(CURVE, scheme, omarlin.deserialize_proof(CURVE, scheme, data)) == data
    if shape == "square":
        g2 = kzg.G2Key(srs, pk.ck.enforced_degree_bounds)
        assert omarlin.verify(pk, [c, d], proof, g2)
        assert not omarlin.verify(pk, [a, a], proof, g2)


def test_golden_file_regenerates():
    import tests_golden
    from golden.make_golden_bls12_377 import CASES
    pinned = json.load(open(os.path.join(HERE, "golden", "marlin_proofs_bls12_377.json")))["cases"]
    assert [c["name"] for c in pinned] == [c["name"] for c in CASES]
    for case, want in zip(CASES, pinned):
        if case["nc"] <= 64:
            assert tests_golden.regenerate_case(case) == want
