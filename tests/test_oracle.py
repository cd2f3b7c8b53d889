"""CPU: the oracle pinned against everything available without the (unbuildable) Rust reference:
known-answer vectors, the reference's own algebraic unit tests re-expressed
(src/ahp/mod.rs:340-387, src/ahp/constraint_systems.rs:309-407), prove/verify acceptance and rejection
(src/test.rs:158-161), the committed golden fixtures, and the C port against the Python specification."""
import hashlib
import json
import os
import random
import struct

import numpy as np
import pytest

import b2m_testutil as util
from oracle import ahp, cport, ec, kzg, marlin, poly as P, r1cs
from oracle import rng as R
from oracle.params import BLS12_381, BN254

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_chacha_known_answers():
    # zero-key keystream heads of ChaCha20 / ChaCha12 / ChaCha8 (eSTREAM / RFC 7539 appendix vectors)
    ks = lambda rounds: struct.pack("<16I", *R.chacha_block([0] * 8, 0, rounds))[:8].hex()
    assert ks(20) == "76b8e0ada0f13d90" and ks(12) == "9bf49a6a0755f953" and ks(8) == "3e00ef2f895f40d6"
    # BlockRng semantics: next_u64 = two consecutive words, low first, across block boundaries
    r = R.ChaChaRng(bytes(32), 20, word_pos=15)
    w = R.chacha_block([0] * 8, 0, 20)[15] | (R.chacha_block([0] * 8, 1, 20)[0] << 32)
    assert r.next_u64() == w and r.word_pos == 17


def test_blake2s_known_answer():
    assert hashlib.blake2s(b"abc", digest_size=32).hexdigest() == "508c5e8c327c14e2e1a72ba34eeb452f37458b209ed63a294d999b4c86675982"


def test_curve_known_answers():
    c = BLS12_381
    two_g = ec.affine_add(c, c.g, c.g)
    assert hex(two_g[0]).startswith("0x572cbea904d67468808c8eb50a9450c9721db309128012543902d0ac358a62ae28f75bb8f1c7c42c39a8c5529bf0f4e")
    for curve in (BLS12_381, BN254):
        assert ec.scalar_mul(curve, curve.fr.p - 1, curve.g) == ec.affine_neg(curve, curve.g)  # group order = |Fr|
        assert ec.on_curve(curve, ec.scalar_mul(curve, 123456789, curve.g))


def test_field_rand_is_montgomery_interpreted():
    f = BLS12_381.fr
    rng = R.test_rng()
    limbs = [R.test_rng().next_u64() for _ in range(1)]
    v = R.field_rand(f, rng)
    raw = R.test_rng()
    attempt = [raw.next_u64() for _ in range(4)]
    attempt[3] &= (1 << 63) - 1
    as_int = sum(l << (64 * i) for i, l in enumerate(attempt))
    if as_int < f.p:
        assert v == f.from_mont(as_int)
    assert limbs[0] == attempt[0]


@pytest.mark.parametrize("log_size", range(1, 10))
def test_domain_unnormalized_bivariate_lagrange_poly(log_size):
    """[reference src/ahp/mod.rs:340-366]"""
    f = BLS12_381.fr
    d = P.Domain(f, 1 << log_size)
    assert ahp.u_h_same_inputs(d) == [ahp.u_h(d, e, e) for e in d.elements()]
    x = R.field_rand(f, R.test_rng())
    assert ahp.u_h_diff_inputs(d, x) == [ahp.u_h(d, x, y) for y in d.elements()]


def test_summation():
    """[reference src/ahp/mod.rs:368-387]: sum over H of p = |H| (a_0 + a_n) for deg p = |H|"""
    f = BLS12_381.fr
    d = P.Domain(f, 16)
    poly = R.poly_rand(f, 16, R.test_rng())
    s = sum(P.evaluate(poly, e, f.p) for e in d.elements()) % f.p
    assert s == (poly[0] + poly[-1]) * 16 % f.p


def test_check_arithmetization():
    """[reference src/ahp/constraint_systems.rs:309-407] with its hand-written 8x8 matrices."""
    f = BLS12_381.fr
    p = f.p
    one = 1
    a = [[(one, 1), (one, 2)], [(one, 3)], [(one, 3)], [(one, 0), (one, 1), (one, 5)], [(one, 1), (one, 2), (one, 6)],
         [(one, 2), (one, 5), (one, 7)], [(one, 3), (one, 4), (one, 6)], [(one, 0), (one, 6), (one, 7)]]
    b = [[], [(one, 1)], [(one, 0)], [(one, 2)], [(one, 3)], [(one, 4)], [(one, 5)], [(one, 6)]]
    c = [[], [(one, 7)], [], [], [], [(one, 3)], [], []]

    class CS:  # just enough of a constraint system for ahp.index
        instance = [1, 0]
        witness = [0] * 6
        num_constraints = 8

        def to_matrices(self):
            return a, b, c

    idx = ahp.index(f, CS())
    dom_h, dom_x = P.Domain(f, 8), P.Domain(f, 2)
    dom_k = P.Domain(f, idx.info.num_non_zero)
    elems = dom_h.elements()
    inverse_map = {e: i for i, e in enumerate(elems)}
    reindexed_inverse = {elems[dom_h.reindex_by_subdomain(dom_x, i)]: i for i in range(8)}
    eq = dict(zip(elems, ahp.u_h_same_inputs(dom_h)))
    polys = {pl.label: pl.coeffs for pl in idx.polys}
    rng = R.test_rng()
    eta = [R.field_rand(f, rng) for _ in range(3)]
    joint = ahp.sum_matrices(a, b, c)
    entry = lambda m, r, col: next((v for v, i in m[r] if i == col), 0)
    for k_index, k in enumerate(dom_k.elements()):
        row_val, col_val = P.evaluate(polys["row"], k, p), P.evaluate(polys["col"], k, p)
        vals = [P.evaluate(polys[l], k, p) for l in ("a_val", "b_val", "c_val")]
        assert idx.evals["row"][k_index] == row_val and idx.evals["col"][k_index] == col_val
        assert [idx.evals[l][k_index] for l in ("val_a", "val_b", "val_c")] == vals
        if k_index < idx.info.num_non_zero:
            col = reindexed_inverse[row_val]
            row = inverse_map[col_val]
            assert col in joint[row]
            lhs = sum(e * v for e, v in zip(eta, vals)) % p
            rhs = pow(eq[row_val], -1, p) * sum(e * entry(m, row, col) for e, m in zip(eta, (a, b, c))) % p
            assert lhs == rhs


SHAPES = [(100, 25), (26, 25), (25, 100), (25, 26), (25, 25)]


@pytest.mark.parametrize("nc,nv", SHAPES[:2] + SHAPES[4:])
@pytest.mark.parametrize("scheme", [kzg.MARLIN, kzg.SONIC])
def test_prove_and_verify_reference_shapes(nc, nv, scheme):
    """[reference src/test.rs:132-203]: verify(prove) == true, verify with a wrong input == false."""
    curve = BLS12_381
    f = curve.fr
    rng = R.test_rng()
    a, b = R.field_rand(f, rng), R.field_rand(f, rng)
    c = a * b % f.p
    d = c * b % f.p
    circ = r1cs.test_circuit(f, a, b, nc, nv)
    srs = marlin.universal_setup(curve, 100, 100, 300, beta=0xabcdef12345, g_scalar=5, gamma=13)
    eng = kzg.Engine(use_trapdoor=True)
    pk = marlin.index(srs, circ, scheme, eng)
    proof = marlin.prove(pk, circ, rng, eng)
    assert marlin.verify(pk, [c, d], proof)
    assert not marlin.verify(pk, [a, a], proof)
    assert len(marlin.serialize_proof(curve, scheme, proof)) == (855 if scheme == kzg.MARLIN else 750)


def test_trapdoor_engine_equals_real_msm_engine():
    curve = BLS12_381
    f = curve.fr
    circ = r1cs.dummy_circuit(f, 3, 4, 10, 16)
    srs = marlin.universal_setup(curve, 16, 16, 48, beta=99991, g_scalar=2, gamma=5)
    outs = []
    for trap in (False, True):
        eng = kzg.Engine(use_trapdoor=trap)
        pk = marlin.index(srs, circ, kzg.MARLIN, eng)
        outs.append((pk.vk_bytes, marlin.serialize_proof(curve, kzg.MARLIN, marlin.prove(pk, circ, R.test_rng(), eng))))
    assert outs[0] == outs[1]


def load_golden():
    with open(os.path.join(GOLDEN, "marlin_proofs.json")) as fh:
        return json.load(fh)


@pytest.mark.parametrize("case", [c["name"] for c in load_golden()["cases"]] if os.path.exists(os.path.join(GOLDEN, "marlin_proofs.json")) else [])
def test_golden_fixtures(case):
    """Committed fixtures (tests/golden/make_golden.py) pin the oracle against silent drift."""
    g = next(c for c in load_golden()["cases"] if c["name"] == case)
    from tests_golden import regenerate_case
    got = regenerate_case(g)
    assert got["vk_sha256"] == g["vk_sha256"] and got["proof_hex"] == g["proof_hex"]


def test_cport_matches_python_oracle():
    rnd = random.Random(4)
    for curve in (BLS12_381, BN254):
        n = 200
        pts = [ec.scalar_mul(curve, rnd.randrange(1, curve.fr.p), curve.g) for _ in range(25)]
        pts = (pts * 8)[:n]
        pts[3] = None
        sc = [rnd.randrange(curve.fr.p) for _ in range(n)]
        sc[0], sc[1], sc[2] = 0, 1, curve.fr.p - 1
        got = util.points_from_limbs(curve, cport.msm(curve.name, util.points_to_limbs(curve, pts), util.fr_to_canon_limbs(curve, sc)))[0]
        assert got == ec.msm_pippenger_arkworks(curve, pts, sc)
        f = curve.fr
        for log_n in (1, 5, 10):
            d = P.Domain(f, 1 << log_n)
            vals = [rnd.randrange(f.p) for _ in range(1 << log_n)]
            buf = util.fr_to_mont_limbs(curve, vals)
            cport.fft(curve.name, buf)
            assert util.fr_from_mont_limbs(curve, buf) == d.fft(vals)
            cport.fft(curve.name, buf, inverse=True)
            assert util.fr_from_mont_limbs(curve, buf) == vals


@pytest.mark.parametrize("curve", [BLS12_381, BN254], ids=lambda c: c.name)
@pytest.mark.parametrize("log_n", [0, 1, 5, 10])
def test_cport_coset_fft_matches_python_oracle(curve, log_n):
    """cport.coset_fft (the checker of the GPU's coset NTTs at sizes Python cannot reach) equals Domain.coset_fft and
    coset_ifft, with 0, 1 and p - 1 among the inputs."""
    f = curve.fr
    rnd = random.Random(40 + log_n)
    n = 1 << log_n
    d = P.Domain(f, n)
    vals = [rnd.randrange(f.p) for _ in range(n)]
    for i, v in zip(range(n), (f.p - 1, 0, 1)):
        vals[-1 - i] = v
    buf = util.fr_to_mont_limbs(curve, vals)
    cport.coset_fft(curve.name, buf)
    assert util.fr_from_mont_limbs(curve, buf) == d.coset_fft(vals)
    buf = util.fr_to_mont_limbs(curve, vals)
    cport.coset_fft(curve.name, buf, inverse=True)
    assert util.fr_from_mont_limbs(curve, buf) == d.coset_ifft(vals)


@pytest.mark.parametrize("case", [c["name"] for c in load_golden()["cases"]] if os.path.exists(os.path.join(GOLDEN, "marlin_proofs.json")) else [])
def test_cpp_prover_reproduces_golden(case):
    """oracle/cport/prover.cpp (the C++ restatement of the reference prover used as CPU baseline) is byte-identical
    to the Python specification on every fixture: index_vk hash, proof bytes and RNG consumption."""
    import hashlib
    import tests_golden as tg
    from marlin_b200 import r1cs as gr1cs
    from oracle.params import CURVES
    g = next(c for c in load_golden()["cases"] if c["name"] == case)
    curve = CURVES[g["curve"]]
    _, a, b, circ, _ = tg.case_inputs(g)
    cs = r1cs.synthesize(curve.fr, circ)
    am, bm, cm = cs.to_matrices()
    nnz = sum(len({i for _, i in ra} | {i for _, i in rb} | {i for _, i in rc}) for ra, rb, rc in zip(am, bm, cm))
    srs = marlin.universal_setup(curve, cs.num_constraints, len(cs.instance) + len(cs.witness), nnz, beta=tg.BETA, g_scalar=tg.G_SCALAR, gamma=tg.GAMMA)
    cid = 0 if g["curve"] == "bls12_381" else 1
    gc = gr1cs.test_circuit(cid, a, b, g["nc"], g["nv"]) if g["circuit"] == "test" else gr1cs.dummy_circuit(cid, a, b, g["nv"], g["nc"])
    H = 1
    while H < gc.num_constraints:
        H *= 2
    K = 1
    while K < nnz:
        K *= 2
    gidx = sorted({0, 1, 2} | {srs.max_degree - d + i for d in (H - 2, K - 2) for i in range(3)})
    pc = "marlin_kzg10" if g["scheme"] == kzg.MARLIN else "sonic_kzg10"
    cp = cport.CpuProver(g["curve"], pc, util.points_to_limbs(curve, srs.powers_of_g), util.points_to_limbs(curve, [srs.power_of_gamma_g(i) for i in gidx]),
                         gidx, gc.num_constraints, gc.num_variables, gc.num_instance, gc.a, gc.b, gc.c)
    try:
        assert hashlib.sha256(cp.vk_bytes).hexdigest() == g["vk_sha256"]
        proof, pos, _ = cp.prove(gc.instance, gc.witness, tg.ZK_SEED, 12, 0)
        assert proof.hex() == g["proof_hex"] and pos == g["zk_rng_word_pos_after"]
    finally:
        cp.close()


@pytest.mark.parametrize("c", [BLS12_381, BN254], ids=lambda c: c.name)
def test_pairing_bilinear_and_nondegenerate(c):
    from oracle import pairing
    pg = pairing.for_curve(c)
    Q = pg.g2_generator()
    assert pg.e12_on_curve(Q) and pg.e12_mul(pg.R, Q) is None
    e1 = pg.pairing(c.g, Q)
    assert e1 != pg.Fq12.one() and e1.pow(pg.R) == pg.Fq12.one()
    a, b = 0x1234567, 0x7654321
    assert pg.pairing(ec.scalar_mul(c, a, c.g), pg.e12_mul(b, Q)) == e1.pow(a * b % pg.R)
    assert pg.pairing_product_is_one([(ec.scalar_mul(c, a, c.g), Q), (ec.affine_neg(c, c.g), pg.e12_mul(a, Q))])
    assert not pg.pairing_product_is_one([(ec.scalar_mul(c, a, c.g), Q), (ec.affine_neg(c, c.g), pg.e12_mul(a + 1, Q))])


@pytest.mark.parametrize("curve", [BLS12_381, BN254], ids=lambda c: c.name)
@pytest.mark.parametrize("scheme", [kzg.MARLIN, kzg.SONIC])
def test_verify_with_real_pairings(scheme, curve):
    """The reference's own acceptance test [src/test.rs:158-161] with `KZG10::check` done by pairings, no trapdoor."""
    f = curve.fr
    rng = R.test_rng()
    a, b = R.field_rand(f, rng), R.field_rand(f, rng)
    c = a * b % f.p
    d = c * b % f.p
    circ = r1cs.test_circuit(f, a, b, 25, 25)
    srs = marlin.universal_setup(curve, 32, 32, 100, beta=0xfeedbeef1234, g_scalar=7, gamma=13)
    eng = kzg.Engine(use_trapdoor=True)
    pk = marlin.index(srs, circ, scheme, eng)
    proof = marlin.prove(pk, circ, rng, eng)
    g2 = kzg.G2Key(srs, pk.ck.enforced_degree_bounds)
    assert marlin.verify(pk, [c, d], proof, g2)
    assert not marlin.verify(pk, [a, a], proof, g2)


@pytest.mark.parametrize("curve", [BLS12_381, BN254], ids=lambda c: c.name)
def test_saved_proof_checker(tmp_path, curve):
    """tests/verify_saved_proof.py (the CPU-side check of `bench.py --save-proof` files) on an oracle-made file:
    accepted as written, rejected after one flipped proof byte."""
    import json
    import verify_saved_proof as vsp
    f = curve.fr
    n = 32
    a, b = 0x1234567890abcdef1234567890abcdef % f.p, 0xfedcba0987654321fedcba0987654321 % f.p
    beta, gamma = 0x5eed5eed5eed5eed5eed5eed, 7
    circ = r1cs.dummy_circuit(f, a, b, 10, n)
    srs = marlin.universal_setup(curve, n, n, 3 * n, beta=beta, g_scalar=1, gamma=gamma)
    eng = kzg.Engine(use_trapdoor=True)
    pk = marlin.index(srs, circ, kzg.MARLIN, eng)
    proof = marlin.serialize_proof(curve, kzg.MARLIN, marlin.prove(pk, circ, R.test_rng(), eng))
    rec = {"curve": curve.name, "pc": "marlin_kzg10", "log_n": 5, "n_gpus": 0, "max_degree": srs.max_degree, "beta": beta, "gamma": gamma,
           "public_input": [str(a * b % f.p)], "proof_hex": proof.hex(), "vk_hex": pk.vk_bytes.hex()}
    path = tmp_path / "proof.json"
    path.write_text(json.dumps(rec))
    res = vsp.verify_file(str(path))
    assert res["ok"] and res["pairing"] and res["num_constraints"] == n
    bad = bytearray(proof)
    bad[-40] ^= 1  # inside the last evaluation / opening data
    rec["proof_hex"] = bytes(bad).hex()
    path.write_text(json.dumps(rec))
    try:
        ok = vsp.verify_file(str(path))["ok"]
    except (ValueError, AssertionError):
        ok = False  # the flipped byte can also make a compressed point undecodable
    assert not ok


def test_compressed_g1_generator_known_answer():
    """ark-serialize compressed form of the BLS12-381 G1 generator: x little-endian with the flags in the two top bits of the last
    byte (bit 7 = y is the larger root, bit 6 = infinity) -- NOT the big-endian zcash encoding (whose first byte would be 0x97).
    The hex string is the value arkworks prints for `G1Affine::prime_subgroup_generator()` (recalled published vector; the oracle's
    format rules themselves are `[U]`, see DESIGN.md section 5)."""
    from oracle import ec, transcript as T
    from oracle.params import BLS12_381 as c
    g = T.g1_compressed(c, c.g)
    assert g.hex() == "bbc622db0af03afbef1a7af93fe8556c58ac1b173f3a4ea105b974974f8c68c30faca94f8c63952694d79731a7d3f117"
    neg = T.g1_compressed(c, ec.affine_neg(c, c.g))
    assert neg[:-1] == g[:-1] and neg[-1] == g[-1] | 0x80  # -G has the larger y
    assert T.g1_compressed(c, None) == bytes(47) + bytes([0x40])
