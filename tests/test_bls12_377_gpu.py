"""GPU: BLS12-377 (curve id 2) end to end -- NTTs and MSMs against the Python model, proof bytes equal to the oracle's and to
the golden file, `Marlin.verify` / `verify_batch` and the oracle's pairing verifier, arkworks SRS and index-key files, and the
Level-1 `commit` / `open_combinations` calls."""
import ctypes
import json
import os
import random

import numpy as np
import pytest

import b2m_testutil as util
import bls12_377_oracle as B
from marlin_b200 import _lib, api, r1cs as gr1cs
from oracle import ec, kzg, marlin as omarlin, r1cs as or1cs
from oracle import rng as orng
from oracle import transcript as T
from oracle.poly import Domain

pytestmark = pytest.mark.gpu
CURVE = B.BLS12_377
CID = _lib.CURVE_BLS12_377
SCHEMES = {"marlin_kzg10": kzg.MARLIN, "sonic_kzg10": kzg.SONIC}
HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "marlin_proofs_bls12_377.json")


@pytest.fixture(scope="module")
def gctx(b2m_ctx):
    c = api.Context.__new__(api.Context)
    c.handle = b2m_ctx
    return c


def gpu_ntt(ctx, vals, log_n, inverse, coset):
    buf = util.fr_to_mont_limbs(CURVE, vals)
    _lib.check(_lib.lib().b2m_ntt(ctx, CID, _lib.ptr(buf), log_n, inverse, coset))
    return buf


# ---- NTT ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("log_n", [4, 5, 8, 10, 12, 20])
def test_ntt_matches_oracle(b2m_ctx, log_n):
    f = CURVE.fr
    n = 1 << log_n
    rnd = random.Random(log_n)
    vals = [rnd.randrange(f.p) for _ in range(n)]
    vals[0], vals[-1] = 0, f.p - 1
    d = Domain(f, n)
    for inverse, coset in ((0, 0), (1, 0), (0, 1), (1, 1)):
        got = util.fr_from_mont_limbs(CURVE, gpu_ntt(b2m_ctx, vals, log_n, inverse, coset))
        want = {(0, 0): d.fft, (1, 0): d.ifft, (0, 1): d.coset_fft, (1, 1): d.coset_ifft}[(inverse, coset)](vals)
        assert got == want, (log_n, inverse, coset)


@pytest.mark.parametrize("log_n", [23, 24])
def test_ntt_large_roundtrip_and_point_check(b2m_ctx, log_n):
    """Sizes the three- and four-pass transforms take: ifft(fft(x)) == x on random input, and on a sparse polynomial the
    forward and coset outputs equal p(w^k) and p(g w^k) (Horner in Python) at scattered k."""
    L = _lib.lib()
    f = CURVE.fr
    n = 1 << log_n
    rng = np.random.default_rng(log_n)
    buf = rng.integers(0, 1 << 63, size=(n, 4), dtype=np.uint64)
    buf[:, 3] &= np.uint64((1 << 59) - 1)  # < 2^251 < r
    orig = buf.copy()
    for coset in (0, 1):
        _lib.check(L.b2m_ntt(b2m_ctx, CID, _lib.ptr(buf), log_n, 0, coset))
        assert not np.array_equal(buf, orig)
        _lib.check(L.b2m_ntt(b2m_ctx, CID, _lib.ptr(buf), log_n, 1, coset))
        assert np.array_equal(buf, orig)
    d = Domain(f, n)
    idx, cv = [0, 5, n // 2 + 1, n - 1], [7, 11, f.p - 1, 13]
    for coset, shift in ((0, 1), (1, f.generator)):
        sp = np.zeros((n, 4), dtype=np.uint64)
        for i, c in zip(idx, cv):
            sp[i] = _lib.ints_to_limbs([f.to_mont(c)], 4)[0]
        _lib.check(L.b2m_ntt(b2m_ctx, CID, _lib.ptr(sp), log_n, 0, coset))
        for k in (0, 1, 2, n // 2, n // 2 + 3, n - 1, 1234567 % n):
            x = shift * d.element(k) % f.p
            want = sum(c * pow(x, i, f.p) for i, c in zip(idx, cv)) % f.p
            assert f.from_mont(_lib.limbs_to_ints(sp[k])[0]) == want, (coset, k)


def test_ntt_above_the_two_adicity_is_rejected(b2m_ctx):
    buf = np.zeros((1, 4), dtype=np.uint64)
    assert _lib.lib().b2m_ntt(b2m_ctx, CID, _lib.ptr(buf), 48, 0, 0) != 0


# ---- MSM ---------------------------------------------------------------------------------------------------------------

def make_srs(ctx, powers, window_bits=0, window_tables=0):
    h = ctypes.c_void_p()
    _lib.check(_lib.lib().b2m_srs_create_layout(ctx, CID, _lib.ptr(powers), len(powers), None, None, 0, window_bits, window_tables,
                                                ctypes.byref(h)))
    return h


def msm_cases(r, N, rnd):
    return [(0, [rnd.randrange(r) for _ in range(N)]), (0, [0] * 200), (3, [1] * 300), (0, [r - 1] * 64),
            (N // 3, [0, 1, r - 1] + [rnd.randrange(r) for _ in range(997)]), (N - 1, [rnd.randrange(r)])]


def test_msm_matches_trapdoor(b2m_ctx):
    rnd = random.Random(1)
    r = CURVE.fr.p
    beta = rnd.randrange(1, r)
    N = 3000
    powers = util.gpu_powers(b2m_ctx, CURVE, CURVE.g, beta, N)
    assert util.points_from_limbs(CURVE, powers[:20]) == ec.fixed_base_powers(CURVE, CURVE.g, beta, 20)
    srs = make_srs(b2m_ctx, powers)
    try:
        for off, sc in msm_cases(r, N, rnd):
            assert util.srs_msm(srs, CURVE, off, sc) == util.trapdoor_msm(CURVE, CURVE.g, beta, off, sc), (off, len(sc))
    finally:
        _lib.lib().b2m_srs_destroy(srs)


def test_msm_duplicate_bases_against_oracle(b2m_ctx):
    """b2m_msm_g1 over arbitrary bases: repeated points, a point next to its negation, infinity"""
    rnd = random.Random(2)
    r = CURVE.fr.p
    P = [ec.scalar_mul(CURVE, rnd.randrange(1, r), CURVE.g) for _ in range(5)]
    bases = [P[0]] * 40 + [P[1], ec.affine_neg(CURVE, P[1])] * 10 + P + [None] * 3 + [P[2]] * 7
    sc = [rnd.randrange(r) for _ in bases]
    sc[:3] = [r - 1, 1, 0]
    out = np.zeros(12, dtype=np.uint64)
    inf = ctypes.c_int()
    _lib.check(_lib.lib().b2m_msm_g1(b2m_ctx, CID, _lib.ptr(util.points_to_limbs(CURVE, bases)), _lib.ptr(util.fr_to_canon_limbs(CURVE, sc)),
                                     len(bases), _lib.ptr(out), ctypes.byref(inf)))
    assert util.points_from_limbs(CURVE, out)[0] == ec.msm_naive(CURVE, bases, sc)


@pytest.mark.parametrize("c,T", [(8, 1), (11, 2), (16, 1), (16, 2)])
def test_msm_reduced_tables_and_bounded_passes(b2m_ctx, monkeypatch, c, T):
    rnd = random.Random(c * 10 + T)
    r = CURVE.fr.p
    beta = rnd.randrange(1, r)
    N = 3000
    powers = util.gpu_powers(b2m_ctx, CURVE, CURVE.g, beta, N)
    monkeypatch.setenv("B2M_MSM_MAX_PAIRS", "700")
    srs = make_srs(b2m_ctx, powers, c, T)
    try:
        W = (CURVE.fr.bits + 1 + c - 1) // c
        m = -(-W // T)
        assert _lib.lib().b2m_srs_window_tables(srs) == -(-W // m)
        for off, sc in msm_cases(r, N, rnd):
            assert util.srs_msm(srs, CURVE, off, sc) == util.trapdoor_msm(CURVE, CURVE.g, beta, off, sc), (off, len(sc))
    finally:
        _lib.lib().b2m_srs_destroy(srs)


# ---- proofs ------------------------------------------------------------------------------------------------------------

def gpu_proof_on_oracle_srs(ctx, scheme, osrs, bounds, gcirc, zk_seed):
    """(index vk bytes, proof bytes) of the GPU on the oracle's SRS"""
    m = api.Marlin("bls12_377", scheme, ctx=ctx)
    gidx = {0, 1, 2}
    if scheme == "sonic_kzg10":
        gidx |= {osrs.max_degree - d + i for d in bounds for i in range(3)}
    gidx = sorted(gidx)
    srs = m.srs_from_points(util.points_to_limbs(CURVE, osrs.powers_of_g), util.points_to_limbs(CURVE, [osrs.power_of_gamma_g(i) for i in gidx]),
                            gidx, 0)
    try:
        pk = m.index(srs, gcirc)
        try:
            return pk.vk_bytes, m.prove(pk, gcirc, api.ZkRng(zk_seed, 12))
        finally:
            pk.close()
    finally:
        srs.close()


def oracle_and_gpu_proof(ctx, scheme, ocirc, gcirc, public_input, zk_seed=bytes(range(32)), beta=0x1234567):
    """(GPU proof bytes, oracle proof bytes) of one circuit on the same SRS and RNG streams; also checks the index vk
    bytes and the oracle's verdicts"""
    f = CURVE.fr
    cs = or1cs.synthesize(f, ocirc)
    nnz = sum(len(set(i for _, i in ra) | set(i for _, i in rb) | set(i for _, i in rc)) for ra, rb, rc in zip(*cs.to_matrices()))
    osrs = omarlin.universal_setup(CURVE, cs.num_constraints, len(cs.instance) + len(cs.witness), nnz, beta=beta, g_scalar=3, gamma=11)
    eng = kzg.Engine(use_trapdoor=True)
    opk = omarlin.index(osrs, ocirc, SCHEMES[scheme], eng)
    oproof = omarlin.prove(opk, ocirc, orng.ChaChaRng(zk_seed, 12), eng)
    assert omarlin.verify(opk, public_input, oproof)
    assert not omarlin.verify(opk, [(x + 1) % f.p for x in public_input], oproof)
    vk_bytes, gbytes = gpu_proof_on_oracle_srs(ctx, scheme, osrs, opk.ck.enforced_degree_bounds, gcirc, zk_seed)
    assert vk_bytes == opk.vk_bytes
    return gbytes, omarlin.serialize_proof(CURVE, SCHEMES[scheme], oproof)


# the reference's test.rs shapes: (num_constraints, num_variables)
REF_SHAPES = {"tall_big": (100, 25), "tall_small": (26, 25), "squat_big": (25, 100), "squat_small": (25, 26), "square": (25, 25)}


@pytest.mark.parametrize("shape", list(REF_SHAPES))
@pytest.mark.parametrize("scheme", list(SCHEMES))
def test_reference_shapes_match_oracle(gctx, shape, scheme):
    f = CURVE.fr
    nc, nv = REF_SHAPES[shape]
    rng = orng.test_rng()
    a, b = orng.field_rand(f, rng), orng.field_rand(f, rng)
    c = a * b % f.p
    d = c * b % f.p
    got, want = oracle_and_gpu_proof(gctx, scheme, or1cs.test_circuit(f, a, b, nc, nv), gr1cs.test_circuit(CID, a, b, nc, nv), [c, d])
    assert got == want


@pytest.mark.parametrize("log_n", [4, 8, 10])
@pytest.mark.parametrize("scheme", list(SCHEMES))
def test_dummy_circuit_matches_oracle(gctx, log_n, scheme):
    f = CURVE.fr
    rng = orng.test_rng()
    a, b = orng.field_rand(f, rng), orng.field_rand(f, rng)
    n = 1 << log_n
    got, want = oracle_and_gpu_proof(gctx, scheme, or1cs.dummy_circuit(f, a, b, 10, n), gr1cs.dummy_circuit(CID, a, b, 10, n), [a * b % f.p])
    assert got == want


def test_golden_file(gctx):
    """the oracle's proofs pinned in tests/golden/marlin_proofs_bls12_377.json (make_golden_bls12_377.py), made on the GPU"""
    import hashlib
    import tests_golden as golden
    cases = json.load(open(GOLDEN))["cases"]
    assert len(cases) >= 5
    for case in cases:
        curve, a, b, ocirc, pub = golden.case_inputs(case)
        assert curve is CURVE
        f = curve.fr
        cs = or1cs.synthesize(f, ocirc)
        nnz = sum(len(set(i for _, i in ra) | set(i for _, i in rb) | set(i for _, i in rc)) for ra, rb, rc in zip(*cs.to_matrices()))
        osrs = omarlin.universal_setup(CURVE, cs.num_constraints, len(cs.instance) + len(cs.witness), nnz, beta=golden.BETA,
                                       g_scalar=golden.G_SCALAR, gamma=golden.GAMMA)
        assert osrs.max_degree == case["srs_max_degree"]
        bounds = omarlin.index(osrs, ocirc, case["scheme"], kzg.Engine(use_trapdoor=True)).ck.enforced_degree_bounds
        if case["circuit"] == "test":
            gcirc = gr1cs.test_circuit(CID, a, b, case["nc"], case["nv"])
        else:
            gcirc = gr1cs.dummy_circuit(CID, a, b, case["nv"], case["nc"])
        vk_bytes, proof = gpu_proof_on_oracle_srs(gctx, case["scheme"], osrs, bounds, gcirc, golden.ZK_SEED)
        assert hashlib.sha256(vk_bytes).hexdigest() == case["vk_sha256"], case["name"]
        assert proof.hex() == case["proof_hex"], case["name"]


@pytest.mark.parametrize("log_n", [12, 20])
def test_large_proof_verifies_on_gpu_and_with_oracle_pairings(gctx, log_n):
    f = CURVE.fr
    n = 1 << log_n
    a, b = 0x1234567890abcdef1234567890abcdef, 0xfedcba0987654321fedcba0987654321
    beta, gamma = 0x5eed5eed5eed5eed5eed5eed, 7
    m = api.Marlin("bls12_377", "marlin_kzg10", ctx=gctx)
    srs = m.universal_setup(n, n, 3 * n, beta=beta, gamma=gamma)
    circ = gr1cs.dummy_circuit(CID, a, b, 10, n)
    handles = []
    try:
        pk = m.index(srs, circ)
        handles.append(pk)
        proof_bytes = m.prove(pk, circ, api.ZkRng.test_rng())
        c_pub = a * b % f.p
        vk = m.verifier_key(pk, srs)
        handles.append(vk)
        assert m.verify(vk, [c_pub], proof_bytes, api.ZkRng(bytes([3]) * 32, 20))
        assert not m.verify(vk, [(c_pub + 1) % f.p], proof_bytes, api.ZkRng(bytes([3]) * 32, 20))
        comms = util.points_from_limbs(CURVE, pk.index_comms)
        lazy = kzg.UniversalParams(CURVE, srs.max_degree, beta, CURVE.g, gamma, powers_of_g="lazy")
        ovk = omarlin.verifier_key_from_public(CURVE, kzg.MARLIN, lazy, n, n, 3 * (n - 1), comms)
        assert ovk.vk_bytes == pk.vk_bytes
        proof = omarlin.deserialize_proof(CURVE, kzg.MARLIN, proof_bytes)
        g2 = kzg.G2Key(lazy, ovk.ck.enforced_degree_bounds)
        assert omarlin.verify(ovk, [c_pub], proof, g2)
        assert not omarlin.verify(ovk, [(c_pub + 1) % f.p], proof, g2)
    finally:
        for h in reversed(handles):
            h.close()
        srs.close()


@pytest.mark.parametrize("scheme", list(SCHEMES))
def test_verify_batch_isolates_the_corrupted_proof(gctx, scheme):
    f = CURVE.fr
    n = 64
    rng = orng.test_rng()
    a, b = orng.field_rand(f, rng), orng.field_rand(f, rng)
    m = api.Marlin("bls12_377", scheme, ctx=gctx)
    md = api.max_degree(n, n, 3 * n)
    bounds = [(1 << k) - 2 for k in range(2, md.bit_length() + 1) if (1 << k) - 2 <= md]
    srs = m.srs_from_trapdoor(md, beta=0x1234567, gamma=7, degree_bounds=bounds)
    circ = gr1cs.dummy_circuit(CID, a, b, 10, n)
    pk = m.index(srs, circ)
    vk = m.verifier_key(pk, srs)
    try:
        distinct = [m.prove(pk, circ, api.ZkRng(bytes([i]) * 32, 12)) for i in range(8)]
        proofs = [distinct[i % 8] for i in range(64)]
        bad = omarlin.deserialize_proof(CURVE, SCHEMES[scheme], proofs[37])
        bad.evaluations[2] = (bad.evaluations[2] + 1) % f.p
        proofs[37] = omarlin.serialize_proof(CURVE, SCHEMES[scheme], bad)
        public = circ.public_input()
        want = [i != 37 for i in range(64)]
        for seed in (1, 2):
            assert m.verify_batch(vk, [public] * 64, proofs, api.ZkRng(bytes([seed]) * 32, 20)) == want
    finally:
        vk.close()
        pk.close()
        srs.close()


# ---- files -------------------------------------------------------------------------------------------------------------

def test_srs_file_roundtrip_and_rejections(gctx, tmp_path):
    m = api.Marlin("bls12_377", "sonic_kzg10", ctx=gctx)
    md = 200
    srs = m.srs_from_trapdoor(md, beta=0xabcdef12345, gamma=7, degree_bounds=[4, 30])
    path = os.path.join(tmp_path, "srs.bin")
    try:
        srs.save_ark(path, compressed=True, degree_bounds=[4, 30])
        blob = open(path, "rb").read()
        for compressed in (True, False):
            loaded = m.load_ark_srs(path, compressed=True, degree_bounds=[4, 30])
            try:
                assert np.array_equal(loaded.powers_limbs, srs.powers_limbs)
                other = os.path.join(tmp_path, "other.bin")
                loaded.save_ark(other, compressed=compressed)
                again = m.load_ark_srs(other, compressed=compressed)
                back = os.path.join(tmp_path, "back.bin")
                again.save_ark(back, compressed=True)
                again.close()
                assert open(back, "rb").read() == blob
            finally:
                loaded.close()
    finally:
        srs.close()
    nb = 48
    rnd = random.Random(4)
    raw = None
    while raw is None:
        x = rnd.randrange(B.Q_MOD)
        y = B.fq_sqrt(x ** 3 + 1)
        raw = (x, y) if y else None
    tors, P, k = None, raw, B.R_MOD
    while k:  # r * raw: a point of the cofactor's torsion
        if k & 1:
            tors = ec.affine_add(CURVE, tors, P)
        P, k = ec.affine_add(CURVE, P, P), k >> 1
    assert tors is not None
    x_off = next(x for x in range(2, 100) if B.fq_sqrt(x ** 3 + 1) is None)
    plants = {
        "both flag bits set": bytes(nb - 1) + b"\xc0",
        "x is not below the field modulus": B.Q_MOD.to_bytes(nb, "little"),
        "not on the curve": x_off.to_bytes(nb, "little"),
        "not in the prime-order subgroup": T.g1_compressed(CURVE, tors),
    }
    for i, (reason, pt) in enumerate(list(plants.items()) + [("not in the prime-order subgroup", T.g1_compressed(CURVE, (0, 1))),
                                                             ("not in the prime-order subgroup", T.g1_compressed(CURVE, (0, B.Q_MOD - 1)))]):
        k = 5 + 17 * i
        data = bytearray(blob)
        data[8 + k * nb:8 + (k + 1) * nb] = pt
        bad = os.path.join(tmp_path, "bad.bin")
        with open(bad, "wb") as fh:
            fh.write(data)
        with pytest.raises(_lib.B2MError) as e:
            m.load_ark_srs(bad, compressed=True)
        assert e.value.code == _lib.ERR_SERIALIZATION
        assert "powers_of_g[%d]: %s" % (k, reason) in str(e.value)


@pytest.mark.parametrize("scheme", list(SCHEMES))
def test_index_key_file_roundtrip_proves_the_same(gctx, tmp_path, scheme):
    f = CURVE.fr
    n = 256
    rng = orng.test_rng()
    a, b = orng.field_rand(f, rng), orng.field_rand(f, rng)
    m = api.Marlin("bls12_377", scheme, ctx=gctx)
    srs = m.universal_setup(n, n, 3 * n, beta=0x77, gamma=5, degree_bounds=(n - 2, 4 * n - 2))
    circ = gr1cs.dummy_circuit(CID, a, b, 10, n)
    handles = []
    try:
        pk = m.index(srs, circ)
        handles.append(pk)
        path = os.path.join(tmp_path, "pk.bin")
        pk.save(path, compressed=True)
        pk2 = m.load_index(srs, path, compressed=True, check_commitments=True)
        handles.append(pk2)
        assert pk2.vk_bytes == pk.vk_bytes
        assert m.prove(pk2, circ, api.ZkRng.test_rng()) == m.prove(pk, circ, api.ZkRng.test_rng())
        vk_path = os.path.join(tmp_path, "vk.bin")
        pk.save_verifier_key(vk_path, compressed=True)
        vk = m.load_verifier_key(vk_path, compressed=True)
        handles.append(vk)
        proof = m.prove(pk, circ, api.ZkRng(bytes([9]) * 32, 12))
        assert m.verify_batch(vk, [circ.public_input()] * 2, [proof, proof], api.ZkRng(bytes([5]) * 32, 20)) == [True, True]
    finally:
        for h in reversed(handles):
            h.close()
        srs.close()


# ---- Level 1 -----------------------------------------------------------------------------------------------------------

def level1_polys(f, rnd):
    return [kzg.LabeledPoly("a", [rnd.randrange(f.p) for _ in range(20)], None, 1), kzg.LabeledPoly("b", [rnd.randrange(f.p) for _ in range(11)], 10, 1),
            kzg.LabeledPoly("c", [0, 0, 5] + [rnd.randrange(f.p) for _ in range(30)], 40, None),
            kzg.LabeledPoly("d", [rnd.randrange(f.p) for _ in range(64)], None, None)]


@pytest.mark.parametrize("scheme", list(SCHEMES))
def test_level1_commit_and_open_match_oracle(gctx, scheme):
    """`PC::commit` and `PC::open` (the one-point `open_combinations`) against the oracle: same commitments, blinding
    polynomials and RNG consumption; same witness commitment and random_v"""
    f = CURVE.fr
    rnd = random.Random(17)
    D = 63
    osrs = kzg.UniversalParams(CURVE, D, 0xabcdef, ec.scalar_mul(CURVE, 3, CURVE.g), 11)
    bounds = [10, 40]
    ck = kzg.CommitterKey(osrs, D, 1, bounds, SCHEMES[scheme])
    polys = level1_polys(f, rnd)
    zk = orng.ChaChaRng(bytes(range(32)), 12)
    eng = kzg.Engine(False)
    ocomms, orands = kzg.commit(eng, ck, polys, zk)
    m = api.Marlin("bls12_377", scheme, ctx=gctx)
    gidx = sorted({0, 1, 2} | ({D - d + i for d in bounds for i in range(3)} if scheme == "sonic_kzg10" else set()))
    srs = m.srs_from_points(util.points_to_limbs(CURVE, osrs.powers_of_g), util.points_to_limbs(CURVE, [osrs.power_of_gamma_g(i) for i in gidx]), gidx)
    try:
        grng = api.ZkRng(bytes(range(32)), 12)
        gpolys = [(util.fr_to_mont_limbs(CURVE, p.coeffs), p.degree_bound, p.hiding_bound) for p in polys]
        comm, shifted, rand, srand = m.commit(srs, gpolys, grng)
        assert grng.word_pos == zk.word_pos
        assert util.points_from_limbs(CURVE, comm) == [c.comm for c in ocomms]
        for i, (c, r) in enumerate(zip(ocomms, orands)):
            assert util.fr_from_mont_limbs(CURVE, rand[i])[:len(r.rand)] == r.rand
            if scheme == "marlin_kzg10":
                assert util.points_from_limbs(CURVE, shifted[i:i + 1])[0] == c.shifted
        z, xi = rnd.randrange(f.p), rnd.randrange(1 << 128)
        ow, orv = kzg.open_at_point(eng, ck, polys, orands, z, lambda k: pow(xi, k, f.p))
        rands = np.zeros((len(polys), 4, 4), dtype=np.uint64)
        srands = np.zeros((len(polys), 4, 4), dtype=np.uint64)
        for i, r in enumerate(orands):
            if r.rand:
                rands[i, :len(r.rand)] = util.fr_to_mont_limbs(CURVE, r.rand)
            if r.shifted_rand:
                srands[i, :len(r.shifted_rand)] = util.fr_to_mont_limbs(CURVE, r.shifted_rand)
        gw, grv = m.open(srs, gpolys, rands, srands, util.fr_to_mont_limbs(CURVE, [z])[0], util.fr_to_mont_limbs(CURVE, [xi])[0],
                         max_degree_bound=max(bounds))
        assert util.points_from_limbs(CURVE, gw)[0] == ow
        assert (None if grv is None else util.fr_from_mont_limbs(CURVE, grv)[0]) == orv
    finally:
        srs.close()
