"""CPU: the Python specification and its C++ restatement (oracle/cport/prover.cpp, the checker the GPU tests use at scale)
on general R1CS -- seeded random satisfiable systems (tests/r1cs_random.py) with 0 to |H|/2 public inputs, several terms
per row, empty A or B rows, hot columns, tall / squat / square shapes and |K| below, equal to and far above |H|.  Until
now both were pinned to each other only on `DummyCircuit` and the reference's test `Circuit`, which have one entry per
row and matrix, three distinct columns and one or two public inputs."""
import numpy as np
import pytest

import b2m_testutil as util
import r1cs_random as R
from marlin_b200 import fields, r1cs as gr1cs
from oracle import cport, kzg, marlin as omarlin, r1cs as or1cs
from oracle import rng as orng
from oracle.params import BLS12_381, BN254

CURVES = {0: BLS12_381, 1: BN254}
SCHEMES = {"marlin_kzg10": kzg.MARLIN, "sonic_kzg10": kzg.SONIC}
ZK_SEED = bytes(range(32))


def _arrays(c):
    return [c.a, c.b, c.c, (c.instance,), (c.witness,)]


@pytest.mark.parametrize("name", list(R.SMALL_CASES))
def test_generator_matches_from_rows(name):
    """The generator's CSR arrays are `from_rows` of its own rows: same input padding, witness shift and squaring; the
    system is satisfied; rows carry no zero coefficient and no column twice, and some rows are not in column order."""
    g = R.small_case(name)
    ref = gr1cs.from_rows(g.curve_id, *g.rows, g.instance, g.witness)
    assert (g.r1cs.num_instance, g.r1cs.num_constraints, g.r1cs.num_variables) == (ref.num_instance, ref.num_constraints, ref.num_variables)
    for got, want in zip(_arrays(g.r1cs), _arrays(ref)):
        for x, y in zip(got, want):
            assert x.dtype == y.dtype and x.shape == y.shape and np.array_equal(x, y)
    assert R.satisfied(g)
    unsorted = 0
    for rows in g.rows:
        for row in rows:
            cols = [i for _, i in row]
            assert len(set(cols)) == len(cols) and all(c % fields.FR_MODULUS[g.curve_id] for c, _ in row)
            unsorted += cols != sorted(cols)
    assert unsorted > 0
    # the oracle's own synthesis of the same circuit gives the same padded system
    cs = or1cs.synthesize(CURVES[g.curve_id].fr, g.circuit(CURVES[g.curve_id].fr))
    assert (len(cs.instance), cs.num_constraints) == (g.X, g.r1cs.num_constraints)
    assert gr1cs.from_rows(g.curve_id, *cs.to_matrices(), cs.instance, cs.witness).instance.tobytes() == g.r1cs.instance.tobytes()


def test_generator_breaks_an_unsatisfied_row():
    """`satisfied` is a real check: one changed witness value breaks it."""
    g = R.generate(0, 5, 2, 30, 10, echo=3, terms=((1, 3), (1, 3), (1, 2)))
    assert R.satisfied(g)
    g.r1cs.witness[3] ^= np.uint64(1)
    assert not R.satisfied(g)


def test_small_cases_cover_the_shapes():
    """The shared small case list covers every class the parity tests are meant to exercise."""
    seen = set()
    for name, spec in R.SMALL_CASES.items():
        g = R.small_case(name)
        a_rows, b_rows, _ = g.rows
        seen |= {("X", g.X), ("shape", R.shape(g)), ("curve", spec["curve"]), ("scheme", spec["scheme"]),
                 ("curve-scheme", spec["curve"], spec["scheme"])}
        if g.X == g.H // 2:
            seen.add(("X", "H/2"))
        seen.add(("K", "<H" if g.K < g.H else ("=H" if g.K == g.H else (">=16H" if g.K >= 16 * g.H else ">H"))))
        if spec.get("columns") == "hot":
            seen.add("hot")
        if any(not r for r in a_rows[:g.live]) and any(not r for r in b_rows[:g.live]):
            seen.add("empty A and B rows")
    for want in [("X", 1), ("X", 2), ("X", 4), ("X", "H/2"), ("K", "<H"), ("K", "=H"), ("K", ">=16H"), ("shape", "tall"),
                 ("shape", "squat"), ("shape", "square"), "hot", "empty A and B rows"]:
        assert want in seen, want
    for c in (0, 1):
        for s in SCHEMES:
            assert ("curve-scheme", c, s) in seen


def oracle_setup(curve, g):
    return omarlin.universal_setup(curve, g.r1cs.num_constraints, g.r1cs.num_variables, g.nnz, beta=0x1234567, g_scalar=3, gamma=11)


def cport_prover(curve, scheme, srs, circ, H, K):
    """CpuProver over the oracle's SRS points (and, for SonicKZG10, the gamma powers of the bounds |H| - 2 and |K| - 2)"""
    gidx = sorted({0, 1, 2} | {srs.max_degree - d + i for d in (H - 2, K - 2) for i in range(3)})
    return cport.CpuProver(curve.name, scheme, util.points_to_limbs(curve, srs.powers_of_g),
                           util.points_to_limbs(curve, [srs.power_of_gamma_g(i) for i in gidx]), gidx,
                           circ.num_constraints, circ.num_variables, circ.num_instance, circ.a, circ.b, circ.c)


@pytest.mark.parametrize("scheme", list(SCHEMES))
@pytest.mark.parametrize("name", list(R.SMALL_CASES))
def test_oracle_and_cport_on_general_r1cs(name, scheme):
    """The oracle proves and verifies the system and rejects the proof when any one public input changes; cport then
    reproduces the oracle's index_vk bytes, both proofs of one continued RNG stream and the stream position exactly."""
    g = R.small_case(name)
    curve = CURVES[g.curve_id]
    f = curve.fr
    circ = g.circuit(f)
    srs = oracle_setup(curve, g)
    eng = kzg.Engine(use_trapdoor=True)
    pk = omarlin.index(srs, circ, SCHEMES[scheme], eng)
    assert pk.index.info.num_non_zero == g.nnz and pk.index.info.num_instance_variables == g.X
    zk = orng.ChaChaRng(ZK_SEED, 12)
    proofs = [omarlin.prove(pk, circ, zk, eng) for _ in range(2)]
    pos = zk.word_pos
    assert omarlin.verify(pk, g.public_input, proofs[0])
    for i in range(len(g.public_input)):
        bad = list(g.public_input)
        bad[i] = (bad[i] + 1) % f.p
        assert not omarlin.verify(pk, bad, proofs[0]), f"accepted with public input {i} changed"
    cp = cport_prover(curve, scheme, srs, g.r1cs, g.H, g.K)
    try:
        assert cp.vk_bytes == pk.vk_bytes
        word = 0
        for proof in proofs:
            got, word, _ = cp.prove(g.r1cs.instance, g.r1cs.witness, ZK_SEED, 12, word)
            assert got == omarlin.serialize_proof(curve, SCHEMES[scheme], proof)
        assert word == pos
    finally:
        cp.close()


def inputs_only_circuit(f, publics):
    """|X| == |H|: public inputs only, no witness -- x_0 * x_1 = x_2 on three inputs, formatted to four variables and
    squared to four constraints"""
    def gen(cs):
        v = [cs.new_input_variable(x) for x in publics]
        cs.enforce_constraint([(1, v[0])], [(1, v[1])], [(1, v[2])])
    return gen


@pytest.mark.parametrize("scheme", list(SCHEMES))
def test_input_length_equal_to_h(scheme):
    """A system whose formatted input fills H (no witness at all) is a valid index in the reference: the indexer only asks
    for a power-of-two input length [reference src/ahp/indexer.rs:192, mod.rs:58-60] and `reindex_by_subdomain` only
    asserts |H| >= |X|.  The oracle proves and verifies it and cport reproduces the bytes."""
    curve = BLS12_381
    f = curve.fr
    publics = [5, 7, 35]
    circ = inputs_only_circuit(f, publics)
    cs = or1cs.synthesize(f, circ)
    assert len(cs.instance) == cs.num_constraints == 4 and not cs.witness
    srs = omarlin.universal_setup(curve, 4, 4, 3, beta=0x1234567, g_scalar=3, gamma=11)
    eng = kzg.Engine(use_trapdoor=True)
    pk = omarlin.index(srs, circ, SCHEMES[scheme], eng)
    zk = orng.ChaChaRng(ZK_SEED, 12)
    proof = omarlin.prove(pk, circ, zk, eng)
    assert omarlin.verify(pk, publics, proof)
    assert not omarlin.verify(pk, [5, 7, 36], proof)
    g = gr1cs.from_rows(0, *cs.to_matrices(), cs.instance, cs.witness)
    cp = cport_prover(curve, scheme, srs, g, 4, 4)
    try:
        assert cp.vk_bytes == pk.vk_bytes
        got, word, _ = cp.prove(g.instance, g.witness, ZK_SEED, 12, 0)
        assert got == omarlin.serialize_proof(curve, SCHEMES[scheme], proof) and word == zk.word_pos
    finally:
        cp.close()
