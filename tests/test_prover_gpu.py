"""GPU parity of the Level-2 ABI (b2m_index_create / b2m_prove) against the oracle: the index
verifier-key bytes and the serialized proof must be BYTE-IDENTICAL to the oracle's on the same SRS,
instance and RNG streams, and the oracle's verifier must accept the GPU proof (and reject it for a
wrong public input), mirroring reference src/test.rs:158-161."""
import numpy as np
import pytest

import b2m_testutil as util
from marlin_b200 import api, r1cs as gr1cs
from oracle import kzg, marlin as omarlin, r1cs as or1cs
from oracle import rng as orng
from oracle.params import BLS12_381, BN254

pytestmark = pytest.mark.gpu

SCHEMES = {"marlin_kzg10": kzg.MARLIN, "sonic_kzg10": kzg.SONIC}


def run_case(ctx, curve, scheme, ocirc, gcirc, public_input, zk_seed=bytes(range(32)), beta=0x1234567, window_bits=0):
    f = curve.fr
    cs = or1cs.synthesize(f, ocirc)
    nnz = sum(len(set(i for _, i in ra) | set(i for _, i in rb) | set(i for _, i in rc)) for ra, rb, rc in zip(*cs.to_matrices()))
    osrs = omarlin.universal_setup(curve, cs.num_constraints, len(cs.instance) + len(cs.witness), nnz, beta=beta, g_scalar=3, gamma=11)
    eng = kzg.Engine(use_trapdoor=True)
    opk = omarlin.index(osrs, ocirc, SCHEMES[scheme], eng)
    zk = orng.ChaChaRng(zk_seed, 12)
    oproof = omarlin.prove(opk, ocirc, zk, eng)
    obytes = omarlin.serialize_proof(curve, SCHEMES[scheme], oproof)
    assert omarlin.verify(opk, public_input, oproof)

    m = api.Marlin(curve.name, scheme, ctx=ctx)
    powers = util.points_to_limbs(curve, osrs.powers_of_g)
    bounds = opk.ck.enforced_degree_bounds
    gidx = [0, 1, 2]
    if scheme == "sonic_kzg10":
        for d in bounds:
            gidx += [osrs.max_degree - d + i for i in range(3)]
    gidx = sorted(set(gidx))
    gam = util.points_to_limbs(curve, [osrs.power_of_gamma_g(i) for i in gidx])
    srs = m.srs_from_points(powers, gam, gidx, window_bits)
    try:
        pk = m.index(srs, gcirc)
        try:
            assert pk.vk_bytes == opk.vk_bytes, "index_vk (ToBytes) differs"
            grng = api.ZkRng(zk_seed, 12)
            gbytes = m.prove(pk, gcirc, grng)
            assert grng.word_pos == zk.word_pos, "zk_rng consumption differs"
            assert gbytes == obytes, "proof bytes differ"
            # a second proof continues the same RNG stream, like the reference's loop (test.rs:138-161)
            oproof2 = omarlin.prove(opk, ocirc, zk, eng)
            assert m.prove(pk, gcirc, grng) == omarlin.serialize_proof(curve, SCHEMES[scheme], oproof2)
            assert not omarlin.verify(opk, [(x + 1) % f.p for x in public_input], oproof)
            return pk.timings()
        finally:
            pk.close()
    finally:
        srs.close()


@pytest.fixture(scope="module")
def gctx(b2m_ctx):
    c = api.Context.__new__(api.Context)
    c.handle = b2m_ctx
    return c


# the reference's own shapes [reference src/test.rs:163-203]: (num_constraints, num_variables)
REF_SHAPES = {"tall_big": (100, 25), "tall_small": (26, 25), "squat_big": (25, 100), "squat_small": (25, 26), "square": (25, 25)}


@pytest.mark.parametrize("shape", list(REF_SHAPES))
@pytest.mark.parametrize("scheme", list(SCHEMES))
def test_reference_test_circuits(gctx, shape, scheme):
    curve = BLS12_381
    nc, nv = REF_SHAPES[shape]
    rng = orng.test_rng()
    a, b = orng.field_rand(curve.fr, rng), orng.field_rand(curve.fr, rng)
    c = a * b % curve.fr.p
    d = c * b % curve.fr.p
    run_case(gctx, curve, scheme, or1cs.test_circuit(curve.fr, a, b, nc, nv), gr1cs.test_circuit(0, a, b, nc, nv), [c, d])


@pytest.mark.parametrize("log_n", [4, 8, 10])
@pytest.mark.parametrize("scheme", list(SCHEMES))
def test_dummy_circuit(gctx, log_n, scheme):
    """BASELINE.json config 1 (2^10, the reference bench's DummyCircuit shape) and smaller."""
    curve = BLS12_381
    n = 1 << log_n
    rng = orng.test_rng()
    a, b = orng.field_rand(curve.fr, rng), orng.field_rand(curve.fr, rng)
    t = run_case(gctx, curve, scheme, or1cs.dummy_circuit(curve.fr, a, b, 10, n), gr1cs.dummy_circuit(0, a, b, 10, n), [a * b % curve.fr.p])
    assert "Marlin::Prover" in t


def test_dense_circuit(gctx):
    """BASELINE.json config 1's "dense" case: seeded random R1CS, 8 non-zeros per row per matrix."""
    curve = BLS12_381
    gen = or1cs.dense_circuit(curve.fr, seed=42, num_constraints=48, num_variables=80, per_row=8)
    cs = or1cs.synthesize(curve.fr, gen)
    a, b, c = or1cs.ConstraintSystem.to_matrices(cs)
    g = gr1cs.from_rows(0, a, b, c, cs.instance, cs.witness)
    run_case(gctx, curve, "marlin_kzg10", gen, g, cs.instance[1:])


@pytest.mark.parametrize("scheme", list(SCHEMES))
def test_bn254(gctx, scheme):
    """BASELINE.json config 4's curve (second field/curve instantiation) at a size the oracle proves in seconds."""
    curve = BN254
    rng = orng.test_rng()
    a, b = orng.field_rand(curve.fr, rng), orng.field_rand(curve.fr, rng)
    run_case(gctx, curve, scheme, or1cs.dummy_circuit(curve.fr, a, b, 10, 64), gr1cs.dummy_circuit(1, a, b, 10, 64), [a * b % curve.fr.p])


def test_error_codes(gctx):
    """Error behaviour mirrors the reference: IndexTooLarge, InstanceDoesNotMatchIndex."""
    from marlin_b200 import _lib
    curve = BLS12_381
    m = api.Marlin("bls12_381", "marlin_kzg10", ctx=gctx)
    srs = m.srs_from_trapdoor(63, beta=5)
    try:
        big = gr1cs.dummy_circuit(0, 3, 4, 10, 64)
        with pytest.raises(_lib.B2MError) as e:
            m.index(srs, big)
        assert e.value.code == 2  # B2M_ERR_INDEX_TOO_LARGE
        small = gr1cs.dummy_circuit(0, 3, 4, 10, 16)
        pk = m.index(srs, small)
        other = gr1cs.dummy_circuit(0, 3, 4, 10, 8)
        with pytest.raises(_lib.B2MError) as e:
            m.prove(pk, other, api.ZkRng.test_rng())
        assert e.value.code == 3  # B2M_ERR_INSTANCE_MISMATCH
        pk.close()
    finally:
        srs.close()


def _golden_cases():
    import json
    import os
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "marlin_proofs.json")
    with open(path) as fh:
        return json.load(fh)["cases"]


@pytest.mark.parametrize("case", _golden_cases(), ids=lambda c: c["name"])
def test_golden_fixture_bytes(gctx, case):
    """The committed fixtures (tests/golden/marlin_proofs.json): GPU-generated SRS, index and proof must
    reproduce sha256(index_vk) and the proof bytes exactly; nothing here reads the oracle's outputs at run time."""
    import hashlib
    import tests_golden as tg
    from oracle import ec
    from oracle.params import CURVES
    curve = CURVES[case["curve"]]
    _, a, b, _, _ = tg.case_inputs(case)
    cid = 0 if case["curve"] == "bls12_381" else 1
    scheme = "marlin_kzg10" if case["scheme"] == kzg.MARLIN else "sonic_kzg10"
    m = api.Marlin(case["curve"], scheme, ctx=gctx)
    g = ec.scalar_mul(curve, tg.G_SCALAR, curve.g)
    circ = gr1cs.test_circuit(cid, a, b, case["nc"], case["nv"]) if case["circuit"] == "test" else gr1cs.dummy_circuit(cid, a, b, case["nv"], case["nc"])
    h = circ.num_constraints
    hs = 1
    while hs < h:
        hs *= 2
    md = case["srs_max_degree"]
    # SonicKZG10 needs the shifted gamma powers of both enforced bounds (|H| - 2, |K| - 2)
    nnz = 3 * (case["nc"] - 1) if case["circuit"] == "dummy" else None
    bounds = [hs - 2]
    ks = 1
    if nnz is None:
        nnz = sum(1 for _ in range(1))  # placeholder, recomputed below
        cs = or1cs.synthesize(curve.fr, tg.case_inputs(case)[3])
        am, bm, cm = cs.to_matrices()
        nnz = sum(len({i for _, i in ra} | {i for _, i in rb} | {i for _, i in rc}) for ra, rb, rc in zip(am, bm, cm))
    while ks < nnz:
        ks *= 2
    bounds.append(ks - 2)
    srs = m.srs_from_trapdoor(md, beta=tg.BETA, g=g, gamma=tg.GAMMA, degree_bounds=bounds)
    try:
        pk = m.index(srs, circ)
        try:
            assert hashlib.sha256(pk.vk_bytes).hexdigest() == case["vk_sha256"]
            rng = api.ZkRng(tg.ZK_SEED, 12)
            assert m.prove(pk, circ, rng).hex() == case["proof_hex"]
            assert rng.word_pos == case["zk_rng_word_pos_after"]
        finally:
            pk.close()
    finally:
        srs.close()


@pytest.mark.parametrize("curve_name,log_n,scheme", [("bls12_381", 16, "marlin_kzg10"), ("bls12_381", 16, "sonic_kzg10"),
                                                     ("bn254", 16, "marlin_kzg10"), ("bls12_381", 20, "marlin_kzg10"),
                                                     ("bn254", 20, "marlin_kzg10"),       # BASELINE.json config 4 at full size
                                                     ("bls12_381", 22, "sonic_kzg10")])   # BASELINE.json config 3 at full size
def test_full_size_proof_verifies(gctx, curve_name, log_n, scheme):
    """Size-independent check at BASELINE.json's sizes (the oracle cannot *prove* 2^20 in reasonable time, but
    verification needs only public data): the GPU proof of a 2^log_n-constraint DummyCircuit is accepted by the
    oracle's restatement of `Marlin::verify` for the right public input and rejected for a wrong one or after a
    one-byte change [reference src/test.rs:158-161]."""
    from oracle import ec
    from oracle.params import CURVES
    curve = CURVES[curve_name]
    f = curve.fr
    n = 1 << log_n
    a, b = 0x1234567890abcdef1234567890abcdef, 0xfedcba0987654321fedcba0987654321
    beta, gamma = 0x5eed5eed5eed5eed5eed5eed, 7
    m = api.Marlin(curve_name, scheme, ctx=gctx)
    srs = m.universal_setup(n, n, 3 * n, beta=beta, gamma=gamma, degree_bounds=(n - 2, 4 * n - 2))
    circ = gr1cs.dummy_circuit(m.curve_id, a, b, 10, n)
    try:
        pk = m.index(srs, circ)
        try:
            proof_bytes = m.prove(pk, circ, api.ZkRng.test_rng())
            comms = util.points_from_limbs(curve, pk.index_comms)
            lazy = kzg.UniversalParams(curve, srs.max_degree, beta, curve.g, gamma, powers_of_g="lazy")
            vk = omarlin.verifier_key_from_public(curve, SCHEMES[scheme], lazy, n, n, 3 * (n - 1), comms)
            assert vk.vk_bytes == pk.vk_bytes
            proof = omarlin.deserialize_proof(curve, SCHEMES[scheme], proof_bytes)
            assert all(ec.on_curve(curve, c.comm) for rnd in proof.commitments for c in rnd)
            c_pub = a * b % f.p
            assert omarlin.verify(vk, [c_pub], proof)
            assert not omarlin.verify(vk, [(c_pub + 1) % f.p], proof)
            # and with the reference's real check: a product of pairings, no trapdoor (oracle/pairing.py, both curves)
            g2 = kzg.G2Key(lazy, vk.ck.enforced_degree_bounds)
            assert omarlin.verify(vk, [c_pub], proof, g2)
            assert not omarlin.verify(vk, [(c_pub + 1) % f.p], proof, g2)
            bad = omarlin.deserialize_proof(curve, SCHEMES[scheme], proof_bytes)
            bad.evaluations[2] = (bad.evaluations[2] + 1) % f.p
            assert not omarlin.verify(vk, [c_pub], bad)
        finally:
            pk.close()
    finally:
        srs.close()


@pytest.mark.parametrize("scheme", list(SCHEMES))
def test_pc_commit_level1(gctx, scheme):
    """Level-1 ABI (b2m_pc_commit) against the oracle's `PC::commit`: same commitments, same blinding polynomials,
    same RNG consumption, for unbounded / bounded / hiding / non-hiding polynomials in one call."""
    import random
    curve = BLS12_381
    f = curve.fr
    rnd = random.Random(17)
    D = 63
    osrs = kzg.UniversalParams(curve, D, 0xabcdef, ec_scalar(curve, 3), 11)
    bounds = [10, 40]
    ck = kzg.CommitterKey(osrs, D, 1, bounds, SCHEMES[scheme])
    polys = [kzg.LabeledPoly("a", [rnd.randrange(f.p) for _ in range(20)], None, 1),
             kzg.LabeledPoly("b", [rnd.randrange(f.p) for _ in range(11)], 10, 1),
             kzg.LabeledPoly("c", [0, 0, 5] + [rnd.randrange(f.p) for _ in range(30)], 40, None),
             kzg.LabeledPoly("d", [rnd.randrange(f.p) for _ in range(64)], None, None),
             kzg.LabeledPoly("e", [7], None, 1)]
    zk = orng.ChaChaRng(bytes(range(32)), 12)
    ocomms, orands = kzg.commit(kzg.Engine(False), ck, polys, zk)
    m = api.Marlin("bls12_381", scheme, ctx=gctx)
    gidx = sorted({0, 1, 2} | ({D - d + i for d in bounds for i in range(3)} if scheme == "sonic_kzg10" else set()))
    srs = m.srs_from_points(util.points_to_limbs(curve, osrs.powers_of_g), util.points_to_limbs(curve, [osrs.power_of_gamma_g(i) for i in gidx]), gidx)
    try:
        grng = api.ZkRng(bytes(range(32)), 12)
        comm, shifted, rand, srand = m.commit(srs, [(util.fr_to_mont_limbs(curve, p.coeffs), p.degree_bound, p.hiding_bound) for p in polys], grng)
        assert grng.word_pos == zk.word_pos
        assert util.points_from_limbs(curve, comm) == [c.comm for c in ocomms]
        for i, (c, r) in enumerate(zip(ocomms, orands)):
            assert util.fr_from_mont_limbs(curve, rand[i])[:len(r.rand)] == r.rand
            if scheme == "marlin_kzg10":
                assert util.points_from_limbs(curve, shifted[i:i + 1])[0] == c.shifted
                if r.shifted_rand:
                    assert util.fr_from_mont_limbs(curve, srand[i])[:len(r.shifted_rand)] == r.shifted_rand
        from marlin_b200 import _lib
        with pytest.raises(_lib.B2MError) as e:
            m.commit(srs, [(util.fr_to_mont_limbs(curve, [1, 2, 3]), None, 1)], None)
        assert e.value.code == 7  # B2M_ERR_MISSING_RNG
    finally:
        srs.close()


def ec_scalar(curve, k):
    from oracle import ec
    return ec.scalar_mul(curve, k, curve.g)


@pytest.mark.parametrize("curve_name,scheme,log_n", [("bls12_381", "marlin_kzg10", 14), ("bls12_381", "sonic_kzg10", 14), ("bn254", "marlin_kzg10", 13),
                                                     ("bn254", "marlin_kzg10", 16), ("bls12_381", "sonic_kzg10", 16),
                                                     ("bls12_381", "marlin_kzg10", 20)])  # BASELINE.json config 2, byte for byte (~3 CPU-minutes)
def test_bytes_match_cpp_cpu_prover(gctx, curve_name, scheme, log_n):
    """Byte-exact parity at sizes the Python oracle cannot prove: the same GPU-generated SRS, the same instance and
    RNG seed go to libb2m (CUDA) and to oracle/cport/prover.cpp (the C++ restatement of the reference prover, itself
    pinned to the Python specification on the golden fixtures); index_vk bytes, proof bytes and the RNG position
    must coincide."""
    from oracle import cport
    n = 1 << log_n
    cid = 0 if curve_name == "bls12_381" else 1
    a, b = 0x1234567890abcdef1234567890abcdef, 0xfedcba0987654321fedcba0987654321
    m = api.Marlin(curve_name, scheme, ctx=gctx)
    srs = m.universal_setup(n, n, 3 * n, beta=0x5eed5eed5eed5eed5eed5eed, gamma=7, degree_bounds=(n - 2, 4 * n - 2))
    circ = gr1cs.dummy_circuit(cid, a, b, 10, n)
    try:
        pk = m.index(srs, circ)
        try:
            # the BASELINE-size case uses bench.py's zk stream (ark_std::test_rng) so that the proof bench.py hashes -- and
            # pins in tests/golden/bench_proof_hashes.json -- is the very proof compared with the C++ prover here
            seed = api.ZkRng.TEST_RNG_SEED if log_n >= 20 else bytes(range(32))
            rng = api.ZkRng(seed, 12)
            gproof = m.prove(pk, circ, rng)
            cp = cport.CpuProver(curve_name, scheme, srs.powers_limbs, srs.gamma_limbs, srs.gamma_indices, circ.num_constraints,
                                 circ.num_variables, circ.num_instance, circ.a, circ.b, circ.c)
            try:
                assert cp.vk_bytes == pk.vk_bytes
                cproof, pos, _ = cp.prove(circ.instance, circ.witness, seed, 12, 0)
                assert cproof == gproof
                assert pos == rng.word_pos
                if log_n >= 20:
                    import hashlib
                    import json
                    import os
                    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bench_proof_hashes.json")) as fh:
                        pinned = json.load(fh)[f"{curve_name}/{scheme}/{log_n}"]
                    assert hashlib.sha256(gproof).hexdigest() == pinned
            finally:
                cp.close()
        finally:
            pk.close()
    finally:
        srs.close()


@pytest.mark.parametrize("scheme", list(SCHEMES))
def test_pc_open_level1(gctx, scheme):
    """Level-1 ABI (b2m_pc_open) against the oracle's `open_individual_opening_challenges` at one point: same
    witness commitment w and same random_v, with bounded / unbounded / hiding / non-hiding polynomials mixed."""
    import random
    curve = BLS12_381
    f = curve.fr
    rnd = random.Random(23)
    D = 63
    osrs = kzg.UniversalParams(curve, D, 0xabcdef, ec_scalar(curve, 3), 11)
    bounds = [10, 40]
    ck = kzg.CommitterKey(osrs, D, 1, bounds, SCHEMES[scheme])
    cases = [
        [kzg.LabeledPoly("a", [rnd.randrange(f.p) for _ in range(20)], None, 1), kzg.LabeledPoly("b", [rnd.randrange(f.p) for _ in range(11)], 10, 1),
         kzg.LabeledPoly("c", [rnd.randrange(f.p) for _ in range(33)], 40, None), kzg.LabeledPoly("d", [rnd.randrange(f.p) for _ in range(64)], None, None)],
        [kzg.LabeledPoly("g", [rnd.randrange(f.p) for _ in range(41)], 40, None), kzg.LabeledPoly("h", [rnd.randrange(f.p) for _ in range(50)], None, None)],
        [kzg.LabeledPoly("k", [rnd.randrange(f.p) for _ in range(9)], None, None)],
    ]
    m = api.Marlin("bls12_381", scheme, ctx=gctx)
    gidx = sorted({0, 1, 2} | ({D - d + i for d in bounds for i in range(3)} if scheme == "sonic_kzg10" else set()))
    srs = m.srs_from_points(util.points_to_limbs(curve, osrs.powers_of_g), util.points_to_limbs(curve, [osrs.power_of_gamma_g(i) for i in gidx]), gidx)
    try:
        for polys in cases:
            zk = orng.ChaChaRng(bytes(range(32)), 12)
            eng = kzg.Engine(False)
            _, orands = kzg.commit(eng, ck, polys, zk)
            z, xi = rnd.randrange(f.p), rnd.randrange(1 << 128)
            ow, orv = kzg.open_at_point(eng, ck, polys, orands, z, lambda k: pow(xi, k, f.p))
            rands = np.zeros((len(polys), 4, 4), dtype=np.uint64)
            srands = np.zeros((len(polys), 4, 4), dtype=np.uint64)
            for i, r in enumerate(orands):
                if r.rand:
                    rands[i, :len(r.rand)] = util.fr_to_mont_limbs(curve, r.rand)
                if r.shifted_rand:
                    srands[i, :len(r.shifted_rand)] = util.fr_to_mont_limbs(curve, r.shifted_rand)
            gw, grv = m.open(srs, [(util.fr_to_mont_limbs(curve, p.coeffs), p.degree_bound, p.hiding_bound) for p in polys], rands, srands,
                             util.fr_to_mont_limbs(curve, [z])[0], util.fr_to_mont_limbs(curve, [xi])[0], max_degree_bound=max(bounds))
            assert util.points_from_limbs(curve, gw)[0] == ow
            assert (None if grv is None else util.fr_from_mont_limbs(curve, grv)[0]) == orv
    finally:
        srs.close()


@pytest.mark.parametrize("scheme", list(SCHEMES))
def test_generic_rng_callback(gctx, scheme):
    """The rng crosses the boundary as a host callback (B2M_RNG_CALLBACK: any `RngCore`, not only ChaCha): a Level-1 commit and
    a whole Level-2 prove driven by a callback over the oracle's generator must give the oracle's bytes and leave the generator
    at the oracle's position -- i.e. the library issues exactly the reference's draws, in its order."""
    curve = BLS12_381
    f = curve.fr
    # Level 1: commit
    import random
    rnd = random.Random(5)
    D = 63
    osrs = kzg.UniversalParams(curve, D, 0xabcdef, ec_scalar(curve, 3), 11)
    bounds = [10, 40]
    ck = kzg.CommitterKey(osrs, D, 1, bounds, SCHEMES[scheme])
    polys = [kzg.LabeledPoly("a", [rnd.randrange(f.p) for _ in range(20)], None, 1), kzg.LabeledPoly("b", [rnd.randrange(f.p) for _ in range(11)], 10, 1),
             kzg.LabeledPoly("c", [rnd.randrange(f.p) for _ in range(30)], 40, None)]
    zk = orng.ChaChaRng(bytes(range(32)), 8)  # ChaCha8: not even one of the fast-path generators of the bench
    ocomms, orands = kzg.commit(kzg.Engine(False), ck, polys, zk)
    m = api.Marlin("bls12_381", scheme, ctx=gctx)
    gidx = sorted({0, 1, 2} | ({D - d + i for d in bounds for i in range(3)} if scheme == "sonic_kzg10" else set()))
    srs = m.srs_from_points(util.points_to_limbs(curve, osrs.powers_of_g), util.points_to_limbs(curve, [osrs.power_of_gamma_g(i) for i in gidx]), gidx)
    try:
        src = orng.ChaChaRng(bytes(range(32)), 8)
        comm, shifted, rand, srand = m.commit(srs, [(util.fr_to_mont_limbs(curve, p.coeffs), p.degree_bound, p.hiding_bound) for p in polys],
                                              api.CallbackRng(src.next_u64))
        assert src.word_pos == zk.word_pos
        assert util.points_from_limbs(curve, comm) == [c.comm for c in ocomms]
        for i, r in enumerate(orands):
            assert util.fr_from_mont_limbs(curve, rand[i])[:len(r.rand)] == r.rand
    finally:
        srs.close()
    # Level 2: prove (the mask polynomial is then drawn on the host through the callback)
    n = 64
    rng = orng.test_rng()
    a, b = orng.field_rand(f, rng), orng.field_rand(f, rng)
    ocirc = or1cs.dummy_circuit(f, a, b, 10, n)
    osrs = omarlin.universal_setup(curve, n, n, 3 * n, beta=0x1234567, g_scalar=1, gamma=7)
    eng = kzg.Engine(use_trapdoor=True)
    opk = omarlin.index(osrs, ocirc, SCHEMES[scheme], eng)
    zk = orng.ChaChaRng(bytes(range(1, 33)), 20)
    want = omarlin.serialize_proof(curve, SCHEMES[scheme], omarlin.prove(opk, ocirc, zk, eng))
    srs = m.srs_from_trapdoor(osrs.max_degree, beta=0x1234567, gamma=7, degree_bounds=(n - 2, 4 * n - 2))
    try:
        gcirc = gr1cs.dummy_circuit(0, a, b, 10, n)
        pk = m.index(srs, gcirc)
        try:
            src = orng.ChaChaRng(bytes(range(1, 33)), 20)
            assert m.prove(pk, gcirc, api.CallbackRng(src.next_u64)) == want
            assert src.word_pos == zk.word_pos
        finally:
            pk.close()
    finally:
        srs.close()


@pytest.mark.parametrize("scheme", list(SCHEMES))
def test_trim_and_open_combinations_level1(gctx, scheme):
    """`PC::trim` + `PC::commit(ck, ..)` + `PC::open_combinations` through the C ABI (b2m_trim, b2m_ck_commit,
    b2m_ck_open_combinations) against the oracle's restatement: same BatchLCProof (w, random_v per point, points in label order),
    the committer key's checks (unsupported bound, degree above the supported one), the MarlinKZG10 shift powers."""
    import random
    from marlin_b200 import _lib
    curve = BLS12_381
    f = curve.fr
    p = f.p
    rnd = random.Random(99)
    D = 63
    osrs = kzg.UniversalParams(curve, D, 0xabcdef, ec_scalar(curve, 3), 11)
    bounds = [10, 40]
    ock = kzg.CommitterKey(osrs, D, 1, bounds, SCHEMES[scheme])
    polys = [kzg.LabeledPoly("a", [rnd.randrange(p) for _ in range(20)], None, 1), kzg.LabeledPoly("b", [rnd.randrange(p) for _ in range(11)], 10, 1),
             kzg.LabeledPoly("c", [rnd.randrange(p) for _ in range(33)], 40, None), kzg.LabeledPoly("d", [rnd.randrange(p) for _ in range(64)], None, None),
             kzg.LabeledPoly("e", [rnd.randrange(p) for _ in range(7)], None, 1)]
    zk = orng.ChaChaRng(bytes(range(32)), 12)
    eng = kzg.Engine(False)
    _, orands = kzg.commit(eng, ock, polys, zk)
    k1, k2, k3 = rnd.randrange(p), rnd.randrange(p), rnd.randrange(p)
    # labels sort as: "b" < "c" < "lc_mixed" < "lc_two": single bounded polynomials, a hiding mix with a constant term, a non-hiding pair
    lcs = [kzg.LinearCombination("b", [(1, "b")]), kzg.LinearCombination("c", [(1, "c")]),
           kzg.LinearCombination("lc_mixed", [(k1, "a"), (k2, "d"), (5, None), (k3, "e")]), kzg.LinearCombination("lc_two", [(k2, "d"), (k1, "d")])]
    z_beta, z_gamma, xi = rnd.randrange(p), rnd.randrange(p), rnd.randrange(1 << 128)
    qs = [("b", ("beta", z_beta)), ("lc_mixed", ("beta", z_beta)), ("lc_two", ("gamma", z_gamma)), ("c", ("gamma", z_gamma)), ("lc_mixed", ("gamma", z_gamma))]
    want = kzg.open_combinations(eng, ock, lcs, polys, orands, qs, xi)
    m = api.Marlin("bls12_381", scheme, ctx=gctx)
    gidx = sorted({0, 1, 2} | ({D - d + i for d in bounds for i in range(3)} if scheme == "sonic_kzg10" else set()))
    srs = m.srs_from_points(util.points_to_limbs(curve, osrs.powers_of_g), util.points_to_limbs(curve, [osrs.power_of_gamma_g(i) for i in gidx]), gidx)
    try:
        ck = m.trim(srs, D, 1, bounds)
        try:
            gp = [(util.fr_to_mont_limbs(curve, q.coeffs), q.degree_bound, q.hiding_bound) for q in polys]
            comm, shifted, rand, srand = m.commit(ck, gp, api.ZkRng(bytes(range(32)), 12))
            label_idx = {q.label: i for i, q in enumerate(polys)}
            lc_idx = {lc.label: i for i, lc in enumerate(lcs)}
            glcs = [[(util.fr_to_mont_limbs(curve, [c])[0], None if t is None else label_idx[t]) for c, t in lc.terms] for lc in lcs]
            gqs = [(lc_idx[l], 0 if pl == "beta" else 1) for l, (pl, _) in qs]
            gctx.profile(True)
            try:
                got = m.open_combinations(ck, gp, rand, srand, glcs, gqs, util.fr_to_mont_limbs(curve, [z_beta, z_gamma]),
                                          util.fr_to_mont_limbs(curve, [xi])[0])
            finally:
                rep = gctx.profile_report()
                gctx.profile(False)
            assert rep["msm_reduce"]["launches"] == 1  # the witness MSMs of both points in one batch
            assert len(got) == len(want) == 2
            for (gw, grv), (ow, orv) in zip(got, want):
                assert util.points_from_limbs(curve, gw)[0] == ow
                assert (None if grv is None else util.fr_from_mont_limbs(curve, grv)[0]) == orv
            if scheme == "marlin_kzg10":
                for d in bounds:
                    assert util.points_from_limbs(curve, ck.shift_power(d))[0] == osrs.powers_of_g[D - d]
            # the committer key's checks [U ark-poly-commit check_degrees_and_bounds / Error::*]
            with pytest.raises(_lib.B2MError) as e:
                m.commit(ck, [(util.fr_to_mont_limbs(curve, [1, 2, 3]), 12, None)], None)  # 12 is not an enforced bound
            assert e.value.code == 1
            with pytest.raises(_lib.B2MError) as e:
                m.open_combinations(ck, gp, rand, srand, [[(util.fr_to_mont_limbs(curve, [2])[0], 1)]], [(0, 0)], util.fr_to_mont_limbs(curve, [z_beta]),
                                    util.fr_to_mont_limbs(curve, [xi])[0])  # a bounded polynomial scaled by 2: EquationHasDegreeBounds
            assert e.value.code == 1
        finally:
            ck.close()
        small = m.trim(srs, 16, 1, [10])
        try:
            with pytest.raises(_lib.B2MError) as e:
                m.commit(small, [(util.fr_to_mont_limbs(curve, list(range(1, 19))), None, None)], None)  # degree 17 > supported 16
            assert e.value.code == 6
        finally:
            small.close()
        with pytest.raises(_lib.B2MError) as e:
            m.trim(srs, D + 1, 1, [])  # TrimmingDegreeTooLarge
        assert e.value.code == 6
    finally:
        srs.close()


def test_destroy_order_is_free(b2m_ctx):
    """Handles may be destroyed in any order: a parent destroyed first is only marked and goes with its last child."""
    curve = BLS12_381
    m = api.Marlin("bls12_381", "marlin_kzg10", device=0)  # its own context, destroyed FIRST
    srs = m.srs_from_trapdoor(63, beta=5)
    circ = gr1cs.dummy_circuit(0, 3, 4, 10, 16)
    pk = m.index(srs, circ)
    ck = m.trim(srs, 63, 1, [10])
    m.ctx.close()
    srs.close()
    proof = m.prove(pk, circ, api.ZkRng.test_rng())  # the index still works: its SRS and context are alive underneath
    assert len(proof) > 800
    ck.close()
    pk.close()


def test_srs_file_save_load(gctx, tmp_path):
    """SURVEY section 8 f-3: an SRS generated on the GPU is written in ark-serialize layout (marlin_b200/srsfile.py), the G1 bytes are
    the oracle's points in `serialize_uncompressed` form, and a key loaded back from the file proves the same bytes."""
    import os
    from marlin_b200 import srsfile
    from oracle import ec
    curve = BLS12_381
    n = 16
    m = api.Marlin("bls12_381", "sonic_kzg10", ctx=gctx)
    beta = 0x1234567
    srs = m.universal_setup(n, n, 3 * n, beta=beta, gamma=7, degree_bounds=(n - 2, 4 * n - 2))
    path = os.path.join(tmp_path, "srs.bin")
    circ = gr1cs.dummy_circuit(0, 3, 4, 10, n)
    try:
        srs.save(path, degree_bounds=(n - 2, 4 * n - 2))
        d = srsfile.read_srs(path)
        nb = curve.fq.nbytes
        want = ec.fixed_base_powers(curve, curve.g, beta, srs.max_degree + 1)
        for i in (0, 1, 2, srs.max_degree):
            x = int.from_bytes(d["powers"][i * 2 * nb:i * 2 * nb + nb], "little")
            y = int.from_bytes(d["powers"][i * 2 * nb + nb:(i + 1) * 2 * nb], "little")
            assert (x, y) == want[i]
        assert sorted(d["neg_powers"]) == sorted(srs.max_degree - b for b in (n - 2, 4 * n - 2))
        pk = m.index(srs, circ)
        proof = m.prove(pk, circ, api.ZkRng.test_rng())
        vk = pk.vk_bytes
        pk.close()
    finally:
        srs.close()
    srs2 = m.load_srs(path)
    try:
        assert srs2.max_degree == 4 * n - 1
        pk = m.index(srs2, circ)
        try:
            assert pk.vk_bytes == vk
            assert m.prove(pk, circ, api.ZkRng.test_rng()) == proof
        finally:
            pk.close()
    finally:
        srs2.close()
