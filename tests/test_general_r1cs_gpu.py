"""GPU byte parity and verification on general R1CS (tests/r1cs_random.py): many public inputs or none, several terms per
row, empty A or B rows, hot or instance-heavy columns, tall / squat / square systems, |K| below and far above |H|.

- small systems: index_vk, two proofs on one continued RNG stream and the stream position equal the Python oracle's;
- at scale: the same against oracle/cport/prover.cpp (pinned to the oracle on these shapes by test_general_r1cs_cpu);
- every proof is accepted by `Marlin.verify_batch` and by the oracle's verifier from public data, and rejected by the
  batch verifier when the first, a middle or the last public input changes;
- edges: |X| == |H| is a valid index; a formatted input that is not a power of two and a column >= num_variables are
  rejected.
A byte mismatch names the first differing proof component (e.g. "round-1 commitment w"), which points at the kernel."""
import time

import pytest

import b2m_testutil as util
import r1cs_random as R
from marlin_b200 import _lib, api, r1cs as gr1cs
from oracle import ahp, cport, kzg, marlin as omarlin, r1cs as or1cs
from oracle import rng as orng
from oracle.params import BLS12_381, BN254

pytestmark = pytest.mark.gpu

CURVES = {0: BLS12_381, 1: BN254}
SCHEMES = {"marlin_kzg10": kzg.MARLIN, "sonic_kzg10": kzg.SONIC}
ZK_SEED = bytes(range(32))
ROUND_LABELS = [["w", "z_a", "z_b", "mask_poly"], ["t", "g_1", "h_1"], ["g_2", "h_2"]]
EVAL_LABELS = ["g_1(beta)", "g_2(gamma)", "t(beta)", "z_b(beta)"]  # sorted by label, as the proof stores them


@pytest.fixture(scope="module")
def gctx(b2m_ctx):
    c = api.Context.__new__(api.Context)
    c.handle = b2m_ctx
    return c


def first_difference(curve, scheme, got, want):
    """name of the first component where two serialized proofs differ (None if equal)"""
    if got == want:
        return None
    try:
        a, b = (omarlin.deserialize_proof(curve, SCHEMES[scheme], x) for x in (got, want))
    except Exception as e:  # noqa: BLE001 -- a framing difference is itself the finding
        return f"proof framing ({type(e).__name__}: {e}; {len(got)} vs {len(want)} bytes)"
    for r, labels in enumerate(ROUND_LABELS):
        for label, x, y in zip(labels, a.commitments[r], b.commitments[r]):
            if x.comm != y.comm:
                return f"round-{r + 1} commitment {label}"
            if x.shifted != y.shifted:
                return f"round-{r + 1} shifted commitment {label}"
    for i, (x, y) in enumerate(zip(a.evaluations, b.evaluations)):
        if x != y:
            return f"evaluation {i} ({EVAL_LABELS[i]})"
    for i, ((w1, v1), (w2, v2)) in enumerate(zip(a.pc_proof, b.pc_proof)):
        if w1 != w2:
            return f"opening proof w at {'beta' if i == 0 else 'gamma'}"
        if v1 != v2:
            return f"opening proof random_v at {'beta' if i == 0 else 'gamma'}"
    return "serialization (components equal, bytes differ)"


def assert_same_proof(curve, scheme, got, want, what="proof"):
    diff = first_difference(curve, scheme, got, want)
    assert diff is None, f"{what} differs first in {diff}"


def test_first_difference_names_the_component():
    """The diagnostics themselves: a changed evaluation or commitment is reported by name."""
    curve = BLS12_381
    g = R.small_case("x4-squat-k-below-h")
    circ = g.circuit(curve.fr)
    srs = omarlin.universal_setup(curve, g.r1cs.num_constraints, g.r1cs.num_variables, g.nnz, beta=0x1234567, g_scalar=3, gamma=11)
    eng = kzg.Engine(use_trapdoor=True)
    pk = omarlin.index(srs, circ, kzg.MARLIN, eng)
    proof = omarlin.prove(pk, circ, orng.ChaChaRng(ZK_SEED, 12), eng)
    good = omarlin.serialize_proof(curve, kzg.MARLIN, proof)
    proof.evaluations[2] = (proof.evaluations[2] + 1) % curve.fr.p
    assert first_difference(curve, "marlin_kzg10", omarlin.serialize_proof(curve, kzg.MARLIN, proof), good) == "evaluation 2 (t(beta))"
    proof.commitments[0][0] = proof.commitments[0][1]
    assert first_difference(curve, "marlin_kzg10", omarlin.serialize_proof(curve, kzg.MARLIN, proof), good) == "round-1 commitment w"
    assert first_difference(curve, "marlin_kzg10", good, good) is None


def gpu_srs_from_oracle(m, curve, scheme, osrs, bounds):
    powers = util.points_to_limbs(curve, osrs.powers_of_g)
    gidx = [0, 1, 2]
    if scheme == "sonic_kzg10":
        gidx += [osrs.max_degree - d + i for d in bounds for i in range(3)]
    gidx = sorted(set(gidx))
    return m.srs_from_points(powers, util.points_to_limbs(curve, [osrs.power_of_gamma_g(i) for i in gidx]), gidx)


def oracle_parity(ctx, curve, scheme, ocirc, gcirc, public_input):
    """`run_case` of test_prover_gpu on any circuit: the GPU's index_vk, two proofs on one continued RNG stream and the
    stream position equal the oracle's; the GPU batch verifier accepts both proofs."""
    f = curve.fr
    cs = or1cs.synthesize(f, ocirc)
    nnz = sum(len(r) for r in ahp.sum_matrices(*cs.to_matrices()))
    osrs = omarlin.universal_setup(curve, cs.num_constraints, len(cs.instance) + len(cs.witness), nnz, beta=0x1234567, g_scalar=3, gamma=11)
    eng = kzg.Engine(use_trapdoor=True)
    opk = omarlin.index(osrs, ocirc, SCHEMES[scheme], eng)
    zk = orng.ChaChaRng(ZK_SEED, 12)
    want = [omarlin.serialize_proof(curve, SCHEMES[scheme], omarlin.prove(opk, ocirc, zk, eng)) for _ in range(2)]
    m = api.Marlin(curve.name, scheme, ctx=ctx)
    srs = gpu_srs_from_oracle(m, curve, scheme, osrs, opk.ck.enforced_degree_bounds)
    try:
        pk = m.index(srs, gcirc)
        try:
            assert pk.vk_bytes == opk.vk_bytes, "index_vk differs"
            grng = api.ZkRng(ZK_SEED, 12)
            got = [m.prove(pk, gcirc, grng) for _ in range(2)]
            for i in range(2):
                assert_same_proof(curve, scheme, got[i], want[i], f"proof {i + 1}")
            assert grng.word_pos == zk.word_pos, "zk_rng consumption differs"
        finally:
            pk.close()
    finally:
        srs.close()
    return want


@pytest.mark.parametrize("scheme", list(SCHEMES))
@pytest.mark.parametrize("name", list(R.SMALL_CASES))
def test_small_general_r1cs_match_oracle(gctx, name, scheme):
    g = R.small_case(name)
    curve = CURVES[g.curve_id]
    oracle_parity(gctx, curve, scheme, g.circuit(curve.fr), g.r1cs, g.public_input)


def _square(n, num_public, live):
    """(live, free, echo) of an n x n system with `num_public` inputs (num_public + 1 a power of two) and `live` rows"""
    return dict(num_public=num_public, live=live, free=n - (num_public + 1) - live, echo=n - live)


# name -> (curve id, PC schemes, generator arguments); |H| and |K| as the comments say
SCALE_CASES = {
    # |X| = 1: division by v_X with stride 1, all witness slots interleaved with x(X) at every point of H
    "no-input": (0, ["marlin_kzg10"], dict(seed=21, terms=(3, 3, 1), **_square(1 << 12, 0, 1 << 11))),           # H 2^12, K 2^15
    "many-inputs": (0, ["sonic_kzg10"], dict(seed=22, terms=(4, 4, 2), **_square(1 << 14, 255, 1 << 13))),     # H 2^14, K 2^18
    "half-inputs": (1, ["marlin_kzg10"], dict(seed=23, terms=(2, 2, 1), columns="instance",
                                              **_square(1 << 12, 2047, 1 << 10))),                            # H 2^12, X 2^11
    "k-below-h": (0, ["sonic_kzg10", "marlin_kzg10"], dict(seed=24, num_public=7, live=1 << 10, free=(1 << 14) - 8 - (1 << 10),
                                                           terms=(2, 2, 1))),                                 # H 2^14, K 2^13
    "k-far-above-h": (0, ["marlin_kzg10"], dict(seed=25, terms=(16, 16, 4), **_square(1 << 12, 15, 1 << 11))),  # H 2^12, K 2^18
    "hot-columns": (1, ["sonic_kzg10"], dict(seed=26, num_public=31, live=1 << 15, free=1 << 13, echo=1 << 15,
                                             terms=((0, 6), (0, 6), (1, 3)), columns="hot", hot=4, hot_share=0.5)),  # tall, H 2^16
    "scale": (0, ["marlin_kzg10"], dict(seed=27, terms=(3, 3, 1), **_square(1 << 18, 1023, 1 << 17))),          # H 2^18, K 2^21
}
SCALE_PARAMS = [(name, scheme) for name, (_, schemes, _) in SCALE_CASES.items() for scheme in schemes]
EXPECT = {"no-input": dict(X=1, H=1 << 12), "many-inputs": dict(X=256, H=1 << 14), "half-inputs": dict(X=2048, H=1 << 12),
          "k-below-h": dict(X=8, H=1 << 14, K=1 << 13), "k-far-above-h": dict(X=16, H=1 << 12, K=1 << 18),
          "hot-columns": dict(X=32, H=1 << 16), "scale": dict(X=1024, H=1 << 18)}


@pytest.mark.parametrize("name,scheme", SCALE_PARAMS, ids=[f"{n}-{s}" for n, s in SCALE_PARAMS])
def test_general_r1cs_at_scale(gctx, name, scheme):
    """GPU against cport at scale (index_vk, proof, RNG position identical), then verification of the GPU proof: the batch
    verifier accepts it and rejects it with the first, a middle or the last public input changed (one batch), and the
    oracle's verifier, given only public data, agrees."""
    cid, _, args = SCALE_CASES[name]
    curve = CURVES[cid]
    f = curve.fr
    t0 = time.time()
    g = R.generate(cid, **args)
    circ = g.r1cs
    for k, v in EXPECT[name].items():
        assert getattr(g, k) == v, (k, getattr(g, k))
    if name == "hot-columns":
        assert R.shape(g) == "tall"
    elif name == "k-below-h":
        assert R.shape(g) == "squat"
    else:
        assert R.shape(g) == "square"
    H, K = g.H, g.K
    beta, gamma = 0x5eed5eed5eed5eed5eed5eed, 7
    m = api.Marlin(curve.name, scheme, ctx=gctx)
    srs = m.universal_setup(circ.num_constraints, circ.num_variables, g.nnz, beta=beta, gamma=gamma, degree_bounds=(H - 2, K - 2))
    try:
        pk = m.index(srs, circ)
        try:
            rng = api.ZkRng(ZK_SEED, 12)
            proof = m.prove(pk, circ, rng)
            t_gpu = time.time() - t0
            cp = cport.CpuProver(curve.name, scheme, srs.powers_limbs, srs.gamma_limbs, srs.gamma_indices, circ.num_constraints,
                                 circ.num_variables, circ.num_instance, circ.a, circ.b, circ.c)
            try:
                assert cp.vk_bytes == pk.vk_bytes, "index_vk differs from cport"
                cproof, pos, _ = cp.prove(circ.instance, circ.witness, ZK_SEED, 12, 0)
            finally:
                cp.close()
            assert_same_proof(curve, scheme, proof, cproof, "GPU proof vs cport")
            assert pos == rng.word_pos, "zk_rng consumption differs from cport"
            t_cport = time.time() - t0 - t_gpu

            pub = g.public_input
            batch_in = [pub]
            if pub:
                for i in sorted({0, len(pub) // 2, len(pub) - 1}):
                    bad = list(pub)
                    bad[i] = (bad[i] + 1) % f.p
                    batch_in.append(bad)
            vk = m.verifier_key(pk, srs)
            try:
                verdicts = m.verify_batch(vk, batch_in, [proof] * len(batch_in), api.ZkRng(bytes([9]) * 32, 20))
            finally:
                vk.close()
            assert verdicts == [True] + [False] * (len(batch_in) - 1), verdicts
            comms = util.points_from_limbs(curve, pk.index_comms)
            lazy = kzg.UniversalParams(curve, srs.max_degree, beta, curve.g, gamma, powers_of_g="lazy")
            ovk = omarlin.verifier_key_from_public(curve, SCHEMES[scheme], lazy, circ.num_constraints, circ.num_variables, g.nnz, comms)
            assert ovk.vk_bytes == pk.vk_bytes
            oproof = omarlin.deserialize_proof(curve, SCHEMES[scheme], proof)
            assert omarlin.verify(ovk, pub, oproof)
            if pub:
                assert not omarlin.verify(ovk, batch_in[-1], oproof)
            print(f"\n{name}/{scheme}: H=2^{H.bit_length() - 1} K=2^{K.bit_length() - 1} X={g.X}: generate+index+prove {t_gpu:.1f} s, "
                  f"cport {t_cport:.1f} s, verify {time.time() - t0 - t_gpu - t_cport:.1f} s")
        finally:
            pk.close()
    finally:
        srs.close()


# ---- edges ------------------------------------------------------------------------------------------------------------
def inputs_only(f, publics):
    def gen(cs):
        v = [cs.new_input_variable(x) for x in publics]
        cs.enforce_constraint([(1, v[0])], [(1, v[1])], [(1, v[2])])
    return gen


@pytest.mark.parametrize("curve_id", [0, 1])
@pytest.mark.parametrize("scheme", list(SCHEMES))
def test_input_length_equal_to_h(gctx, curve_id, scheme):
    """|X| == |H| (public inputs only, no witness) is a valid index in the reference -- the indexer asks only for a
    power-of-two input length [reference src/ahp/indexer.rs:192-194] and `reindex_by_subdomain` for |H| >= |X| -- and the
    oracle and cport prove it (test_general_r1cs_cpu).  The GPU proves the same bytes and its verifier accepts them."""
    curve = CURVES[curve_id]
    f = curve.fr
    publics = [5, 7, 35]
    ocirc = inputs_only(f, publics)
    cs = or1cs.synthesize(f, ocirc)
    assert len(cs.instance) == cs.num_constraints == 4
    gcirc = gr1cs.from_rows(curve_id, *cs.to_matrices(), cs.instance, cs.witness)
    proofs = oracle_parity(gctx, curve, scheme, ocirc, gcirc, publics)
    m = api.Marlin(curve.name, scheme, ctx=gctx)
    srs = m.universal_setup(4, 4, 3, beta=0x1234567, degree_bounds=(2, 2))
    try:
        pk = m.index(srs, gcirc)
        vk = m.verifier_key(pk, srs)
        try:
            proof = m.prove(pk, gcirc, api.ZkRng(ZK_SEED, 12))
            assert len(proof) == len(proofs[0])
            assert m.verify_batch(vk, [publics, [5, 7, 36]], [proof, proof], api.ZkRng(bytes([3]) * 32, 20)) == [True, False]
        finally:
            vk.close()
            pk.close()
    finally:
        srs.close()


def test_rejects_malformed_systems(gctx):
    """A formatted input whose length is not a power of two is the reference's InvalidPublicInputLength on the GPU, the
    oracle and cport alike; a column index >= num_variables is rejected by the index before anything is read through it."""
    curve = BLS12_381
    f = curve.fr
    m = api.Marlin("bls12_381", "marlin_kzg10", ctx=gctx)
    srs = m.srs_from_trapdoor(63, beta=5, degree_bounds=(6, 6))
    try:
        # 3 formatted inputs (no power of two) and one witness, four constraints: x_1 * x_2 = w
        a_rows, b_rows, c_rows = [[(1, 1)], [], [], []], [[(1, 2)], [], [], []], [[(1, 3)], [], [], []]
        good = gr1cs.from_rows(0, a_rows, b_rows, c_rows, [1, 5, 7, 35], [])  # the same rows with an input of four: accepted
        m.index(srs, good).close()
        bad = gr1cs.R1CS(0, 3, good.a, good.b, good.c, good.instance[:3], good.instance[3:])
        with pytest.raises(_lib.B2MError) as e:
            m.index(srs, bad)
        assert e.value.code == 4  # B2M_ERR_INVALID_PUBLIC_INPUT_LEN

        class CS:
            instance, witness, num_constraints = [1, 5, 7], [35], 4

            def to_matrices(self):
                return a_rows, b_rows, c_rows
        with pytest.raises(ValueError, match="InvalidPublicInputLength"):
            ahp.index(f, CS())
        with pytest.raises(RuntimeError, match="code 4"):
            cport.CpuProver("bls12_381", "marlin_kzg10", srs.powers_limbs, srs.gamma_limbs, srs.gamma_indices, 4, 4, 3, bad.a, bad.b, bad.c)

        col = good.c[1].copy()
        col[0] = 4  # == num_variables
        with pytest.raises(_lib.B2MError) as e:
            m.index(srs, gr1cs.R1CS(0, 4, good.a, good.b, (good.c[0], col, good.c[2]), good.instance, good.witness))
        assert e.value.code == 1 and "column index 4 out of range" in str(e.value)
    finally:
        srs.close()
