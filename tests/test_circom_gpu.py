"""GPU: circom circuits (Marlin.load_r1cs / load_wtns / which_is_unsatisfied) on BLS12-381 and BN254.

- parity: tests/r1cs_random.py systems written as circom files load to the arrays `from_rows` makes from the same rows in
  normal form, index to the same vk_bytes, prove the same bytes, verify with the unpadded public signals and reject a
  changed one; one small system also matches the Python oracle and `IndexProverKey.save` bytes;
- normal form: shuffled rows, duplicate wires (wire 0 included), zero coefficients, a row cancelling to nothing and rows of
  2, 33 and 1000+ terms load and prove like their normalised rows;
- chunks: more constraints than one decode chunk, normalised rows on both sides of a boundary, a bad term only in a later
  chunk is the one named;
- corruption: coefficient >= r, wire >= nWires, witness >= r, wtns[0] != 1, a changed witness value;
- a ceremony SRS (load_ptau) proves and verifies a circom circuit;
- at the size users run: bench.py's 2^20 DummyCircuit as circom files loads to `dummy_circuit`'s arrays and proves to the
  pinned hash on both curves."""
import hashlib
import json
import os

import numpy as np
import pytest

import circom_writer as cw
import ptau_writer as pw
import r1cs_random as R
from marlin_b200 import _lib, api, fields, r1cs as gr1cs
from oracle.params import BLS12_381, BN254

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
CURVES = {"bls12_381": BLS12_381, "bn254": BN254}
ZK_SEED = bytes(range(32))


@pytest.fixture(scope="module")
def gctx(b2m_ctx):
    c = api.Context.__new__(api.Context)
    c.handle = b2m_ctx
    return c


def rng():
    return api.ZkRng(bytes([5]) * 32, 20)


def same_arrays(got, want):
    assert got.num_instance == want.num_instance and got.num_constraints == want.num_constraints
    assert got.num_variables == want.num_variables
    for name in "abc":
        for x, y in zip(getattr(got, name), getattr(want, name)):
            assert np.array_equal(np.asarray(x), np.asarray(y)), name
    if got.instance is not None:
        assert np.array_equal(got.instance, want.instance) and np.array_equal(got.witness, want.witness)


def write_pair(tmp_path, cid, n_wires, n_pub_out, n_pub_in, cons, values, name="c"):
    p = fields.FR_MODULUS[cid]
    r = cw.write_r1cs(os.path.join(tmp_path, name + ".r1cs"), p, n_wires, n_pub_out, n_pub_in, cons)
    w = cw.write_wtns(os.path.join(tmp_path, name + ".wtns"), p, values)
    return r, w


def reference(cid, cons, values, ni0):
    """from_rows of the rows in normal form"""
    p = fields.FR_MODULUS[cid]
    rows = [cw.normal_form([[(c, w) for w, c in con[j]] for con in cons], p) for j in range(3)]
    return gr1cs.from_rows(cid, *rows, values[:ni0], values[ni0:])


def prove_both(m, srs, got, want):
    pks = [m.index(srs, got), m.index(srs, want)]
    try:
        assert pks[0].vk_bytes == pks[1].vk_bytes
        proofs = [m.prove(pk, r, api.ZkRng(ZK_SEED, 12)) for pk, r in zip(pks, (got, want))]
        assert proofs[0] == proofs[1]
        return pks, proofs[0]
    except Exception:
        for pk in pks:
            pk.close()
        raise


PARITY = {  # name: curve, generate() arguments
    "no-public-inputs": ("bls12_381", dict(seed=31, num_public=0, live=40, free=23, echo=24, terms=(3, 3, 1))),
    "inputs-cross-pow2": ("bn254", dict(seed=32, num_public=4, live=30, free=20, terms=((1, 4), (1, 4), (1, 3)))),
    "tall-hot": ("bls12_381", dict(seed=33, num_public=2, live=50, free=10, echo=60, terms=((0, 4), (0, 4), (1, 3)), columns="hot")),
    "wide": ("bn254", dict(seed=34, num_public=3, live=12, free=80, terms=(2, 2, 1))),
}


@pytest.mark.parametrize("case", sorted(PARITY))
def test_random_systems_load_like_from_rows_and_prove_the_same_bytes(gctx, tmp_path, case):
    curve_name, spec = PARITY[case]
    m = api.Marlin(curve_name, "marlin_kzg10", ctx=gctx)
    g = R.generate(m.curve_id, keep_rows=True, **spec)
    n_wires, n_out, n_in, cons, values = cw.from_generated(g)
    rp, wp = write_pair(tmp_path, m.curve_id, n_wires, n_out, n_in, cons, values)
    got = m.load_wtns(m.load_r1cs(rp), wp)
    want = reference(m.curve_id, cons, values, 1 + n_out + n_in)
    same_arrays(got, want)
    assert m.which_is_unsatisfied(got) is None and m.which_is_unsatisfied(g.r1cs) is None
    srs = m.universal_setup(got.num_constraints, got.num_variables, 3 * got.num_constraints + 3 * g.nnz, beta=0x5eed, gamma=7)
    try:
        pks, proof = prove_both(m, srs, got, want)
        vk = m.verifier_key(pks[0], srs)
        try:
            assert m.verify(vk, g.public_input, proof, rng())
            if g.public_input:
                bad = list(g.public_input)
                bad[-1] = (bad[-1] + 1) % fields.FR_MODULUS[m.curve_id]
                assert not m.verify(vk, bad, proof, rng())
        finally:
            vk.close()
            for pk in pks:
                pk.close()
    finally:
        srs.close()


def test_small_system_matches_the_oracle_and_saves_the_same_key(gctx, tmp_path):
    curve = BLS12_381
    m = api.Marlin("bls12_381", "marlin_kzg10", ctx=gctx)
    g = R.generate(m.curve_id, keep_rows=True, seed=41, num_public=2, live=20, free=9, terms=(2, 2, 1))
    n_wires, n_out, n_in, cons, values = cw.from_generated(g)
    rp, wp = write_pair(tmp_path, m.curve_id, n_wires, n_out, n_in, cons, values)
    got = m.load_wtns(m.load_r1cs(rp), wp)
    want = reference(m.curve_id, cons, values, 1 + n_out + n_in)
    import test_general_r1cs_gpu as T
    proofs = T.oracle_parity(gctx, curve, "marlin_kzg10", g.circuit(curve.fr), got, g.public_input)
    assert proofs
    # IndexProverKey.save of the loaded matrices equals that of the from_rows index
    srs = m.universal_setup(got.num_constraints, got.num_variables, 6 * got.num_constraints, beta=0x1234567, gamma=11)
    try:
        matrices_only = m.load_r1cs(rp)
        assert matrices_only.instance is None and matrices_only.witness is None
        assert matrices_only.num_variables == got.num_variables
        pks = [m.index(srs, matrices_only), m.index(srs, want)]
        try:
            files = []
            for i, pk in enumerate(pks):
                path = os.path.join(tmp_path, f"pk{i}.bin")
                pk.save(path)
                files.append(open(path, "rb").read())
            assert files[0] == files[1]
        finally:
            for pk in pks:
                pk.close()
    finally:
        srs.close()


def messy_constraints(cid, seed):
    """satisfied constraints with shuffled terms, duplicate wires (wire 0 included), zero coefficients, a row cancelling
    to nothing and rows of 2, 33 and 1200 terms; wires 0 one, 1-2 public, 3.. witnesses"""
    p = fields.FR_MODULUS[cid]
    rnd = np.random.default_rng(seed)
    n_wires = 64
    z = [1] + [int(rnd.integers(1, 1 << 62)) for _ in range(n_wires - 1)]
    cons = []

    def lc(n):
        """n terms over the wires below the outputs; from 5 terms on, wire 0 twice and a zero coefficient among them"""
        if n < 5:
            w = int(rnd.integers(0, 40))
            return [(w, int(rnd.integers(1, 1 << 40))) for _ in range(n)]  # one wire, repeated
        terms = [(int(rnd.integers(0, 40)), int(rnd.integers(0, 1 << 40))) for _ in range(n - 3)]
        terms += [(0, 3), (0, p - 1), (5, 0)]
        return [terms[i] for i in rnd.permutation(len(terms))]

    def value(lc_):
        return sum(c * z[w] for w, c in lc_) % p

    out_wires = list(range(40, 64))
    for k, n in enumerate([2, 33, 1200, 3, 1, 5]):
        a, b = lc(n), lc(max(n // 3, 1))
        ow = out_wires[k]
        cf = lc(2)
        # C = cf + (wire ow) with z[ow] solving the row
        z[ow] = (value(a) * value(b) - value(cf)) % p
        cons.append((a, b, cf + [(ow, 1)]))
    # a row whose A cancels to nothing: (w, 5) + (w, p - 5); B anything, C = 0 written as a zero coefficient
    cons.append(([(7, 5), (7, p - 5)], [(8, 1)], [(9, 0)]))
    return n_wires, cons, z


@pytest.mark.parametrize("curve_name", ["bls12_381", "bn254"])
def test_rows_are_normalised(gctx, tmp_path, curve_name):
    m = api.Marlin(curve_name, "marlin_kzg10", ctx=gctx)
    n_wires, cons, z = messy_constraints(m.curve_id, 51)
    rp, wp = write_pair(tmp_path, m.curve_id, n_wires, 1, 1, cons, z)
    got = m.load_wtns(m.load_r1cs(rp), wp)
    want = reference(m.curve_id, cons, z, 3)
    same_arrays(got, want)
    assert int(got.a[0][7] - got.a[0][6]) == 0  # the row that cancels
    nnz = sum(int(x[0][-1]) for x in (got.a, got.b, got.c))
    srs = m.universal_setup(got.num_constraints, got.num_variables, nnz, beta=0x5eed, gamma=7)
    try:
        pks, _ = prove_both(m, srs, got, want)
        for pk in pks:
            pk.close()
    finally:
        srs.close()


def test_chunks_keep_rows_whole_and_name_the_lowest_bad_term(gctx, tmp_path):
    """2^18 + 2^14 constraints of three one-term LCs (> one 2^18-term chunk): rows with duplicate wires on both sides of the
    first chunk boundary (constraint 87380 starts chunk 2); bad terms only in chunk 4, the lower one named"""
    m = api.Marlin("bn254", "marlin_kzg10", ctx=gctx)
    cid, p = m.curve_id, fields.FR_MODULUS[m.curve_id]
    n = (1 << 18) + (1 << 14)
    n_wires = 8
    z = [1, 6, 2, 3, 2, 2, 2, 2]  # c = a b = 6
    base = ([(2, 1)], [(3, 1)], [(1, 1)])
    cons = [base] * n
    messy = ([(4, 2), (2, p - 1)], [(3, 1)], [(1, 3), (1, p - 2)])  # A = 2a - a = a, C = 3c - 2c = c
    for k in (87379, 87380, 87381, 87382, 200000, n - 1):
        cons[k] = messy
    rp, wp = write_pair(tmp_path, cid, n_wires, 1, 0, cons, z)
    got = m.load_wtns(m.load_r1cs(rp), wp)
    want = reference(cid, cons, z, 2)
    same_arrays(got, want)
    # bad terms: a coefficient >= r in constraint 270000 (chunk 4) and a wire >= nWires in 270001
    bad = list(cons)
    bad[270000] = ([(2, p)], [(3, 1)], [(1, 1)])
    bad[270001] = ([(2, 1)], [(9, 1)], [(1, 1)])
    rp = cw.write_r1cs(os.path.join(tmp_path, "bad.r1cs"), p, n_wires, 1, 0, bad)
    with pytest.raises(_lib.B2MError, match=r"constraints\[270000\]\.A\[0\]: coefficient not below r"):
        m.load_r1cs(rp)
    bad[270000] = base
    rp = cw.write_r1cs(os.path.join(tmp_path, "bad2.r1cs"), p, n_wires, 1, 0, bad)
    with pytest.raises(_lib.B2MError, match=r"constraints\[270001\]\.B\[0\]: wire 9 >= nWires 8"):
        m.load_r1cs(rp)


@pytest.mark.parametrize("curve_name", ["bls12_381", "bn254"])
def test_corruption_is_named(gctx, tmp_path, curve_name):
    m = api.Marlin(curve_name, "marlin_kzg10", ctx=gctx)
    cid, p = m.curve_id, fields.FR_MODULUS[m.curve_id]
    g = R.generate(cid, keep_rows=True, seed=61, num_public=1, live=30, free=12, terms=((1, 4), (1, 4), (1, 3)))
    n_wires, n_out, n_in, cons, values = cw.from_generated(g)
    rp, wp = write_pair(tmp_path, cid, n_wires, n_out, n_in, cons, values)
    r = m.load_r1cs(rp)
    bad = [tuple(list(lc) for lc in con) for con in cons]
    bad[12][2][0] = (bad[12][2][0][0], p + 5)
    with pytest.raises(_lib.B2MError, match=r"constraints\[12\]\.C\[0\]: coefficient not below r"):
        m.load_r1cs(cw.write_r1cs(os.path.join(tmp_path, "b1.r1cs"), p, n_wires, n_out, n_in, bad))
    bad = [tuple(list(lc) for lc in con) for con in cons]
    bad[12][1].append((n_wires + 1, 1))
    i = len(bad[12][1]) - 1
    with pytest.raises(_lib.B2MError, match=rf"constraints\[12\]\.B\[{i}\]: wire {n_wires + 1} >= nWires {n_wires}"):
        m.load_r1cs(cw.write_r1cs(os.path.join(tmp_path, "b2.r1cs"), p, n_wires, n_out, n_in, bad))
    vals = list(values)
    vals[20] = p
    with pytest.raises(_lib.B2MError, match=r"witness\[20\]: not below r"):
        m.load_wtns(r, cw.write_wtns(os.path.join(tmp_path, "w1.wtns"), p, vals))
    vals = list(values)
    vals[0] = 2
    with pytest.raises(ValueError, match=r"witness\[0\] is 2"):
        m.load_wtns(r, cw.write_wtns(os.path.join(tmp_path, "w2.wtns"), p, vals))
    with pytest.raises(ValueError, match="nWitness"):
        m.load_wtns(r, cw.write_wtns(os.path.join(tmp_path, "w3.wtns"), p, values[:-1]))
    other = "bn254" if curve_name == "bls12_381" else "bls12_381"
    with pytest.raises(ValueError, match=f"the {curve_name} scalar field, this Marlin instance is {other}"):
        api.Marlin(other, "marlin_kzg10", ctx=gctx).load_r1cs(rp)
    # a changed witness value: the lowest failing constraint is named, check=False loads
    w = next(w for w, _ in cons[5][2] + cons[5][0] + cons[5][1] if w >= 1 + n_out + n_in)
    vals = list(values)
    vals[w] = (vals[w] + 1) % p
    path = cw.write_wtns(os.path.join(tmp_path, "w4.wtns"), p, vals)
    loose = m.load_wtns(r, path, check=False)
    first = m.which_is_unsatisfied(loose)
    assert first is not None and first <= 5
    with pytest.raises(ValueError, match=rf"constraint {first} is not satisfied"):
        m.load_wtns(r, path)
    # the same row as a Python check of the padded system
    pz = np.array([fields.fr_from_mont(cid, v) for v in _lib.limbs_to_ints(np.concatenate([loose.instance, loose.witness]))], dtype=object)

    def mv(mat):
        row_ptr, col, coeff = mat
        vals_ = [fields.fr_from_mont(cid, v) for v in _lib.limbs_to_ints(coeff)]
        return [sum(vals_[e] * pz[int(col[e])] for e in range(int(row_ptr[k]), int(row_ptr[k + 1]))) % p for k in range(len(row_ptr) - 1)]
    a, b, c = mv(loose.a), mv(loose.b), mv(loose.c)
    assert first == next(k for k in range(len(a)) if a[k] * b[k] % p != c[k])
    # dummy_circuit and from_rows instances hold
    assert m.which_is_unsatisfied(gr1cs.dummy_circuit(cid, 3, 5, 10, 64)) is None
    assert m.which_is_unsatisfied(R.generate(cid, seed=62, num_public=3, live=12, free=12, echo=16, terms=(12, 12, 4)).r1cs) is None


@pytest.mark.parametrize("curve_name", ["bls12_381", "bn254"])
def test_ceremony_srs_proves_a_circom_circuit(gctx, tmp_path, curve_name):
    from marlin_b200 import ptau
    curve = CURVES[curve_name]
    m = api.Marlin(curve_name, "marlin_kzg10", ctx=gctx)
    g = R.generate(m.curve_id, keep_rows=True, seed=71, num_public=2, live=12, free=10, terms=(2, 2, 1))
    n_wires, n_out, n_in, cons, z = cw.from_generated(g)
    rp, wp = write_pair(tmp_path, m.curve_id, n_wires, n_out, n_in, cons, z)
    r = m.load_wtns(m.load_r1cs(rp), wp)
    nnz = sum(int(x[0][-1]) for x in (r.a, r.b, r.c))
    md = api.max_degree(r.num_constraints, r.num_variables, nnz)
    power = ptau.power_for_degree(md)
    path = pw.write(os.path.join(tmp_path, "c.ptau"), pw.sections(curve, power, 0x5eed5eed, 7, 0xbe7a))
    srs = m.load_ptau(path, max_degree=md, rng=rng())
    try:
        pk = m.index(srs, r)
        vk = m.verifier_key(pk, srs)
        try:
            proof = m.prove(pk, r, api.ZkRng.test_rng())
            assert m.verify(vk, z[1:3], proof, rng())
            assert not m.verify(vk, [z[1], z[2] + 1], proof, rng())
        finally:
            vk.close()
            pk.close()
    finally:
        srs.close()


# ---- at the size users run ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("curve_name", ["bls12_381", "bn254"])
def test_bench_dummy_circuit_as_circom_files_proves_the_pinned_hash(gctx, tmp_path, curve_name):
    n = 1 << 20
    m = api.Marlin(curve_name, "marlin_kzg10", ctx=gctx)
    cid = m.curve_id
    a, b = 0x1234567890abcdef1234567890abcdef, 0xfedcba0987654321fedcba0987654321
    rp, wp = os.path.join(tmp_path, "d.r1cs"), os.path.join(tmp_path, "d.wtns")
    cw.dummy_files(rp, wp, cid, a, b, 10, n)
    got = m.load_wtns(m.load_r1cs(rp), wp)
    same_arrays(got, gr1cs.dummy_circuit(cid, a, b, 10, n))
    srs = m.universal_setup(n, n, 3 * n, beta=0x5eed5eed5eed5eed5eed5eed, gamma=7)
    handles = [srs]
    try:
        pk = m.index(srs, got)
        handles.append(pk)
        proof = m.prove(pk, got, api.ZkRng.test_rng())
        with open(os.path.join(HERE, "golden", "bench_proof_hashes.json")) as fh:
            pinned = json.load(fh)[f"{curve_name}/marlin_kzg10/20"]
        assert hashlib.sha256(proof).hexdigest() == pinned
        vk = m.verifier_key(pk, srs)
        handles.append(vk)
        assert m.verify(vk, [a * b % fields.FR_MODULUS[cid]], proof, rng())
    finally:
        for x in handles[::-1]:
            x.close()
