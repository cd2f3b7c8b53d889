"""GPU: batched `Marlin::verify` (b2m_vk_create / b2m_verify_batch, marlin_b200.api.Marlin.verify*) on both curves and both PC
schemes -- GPU proofs, the oracle's golden proofs and the replay kit accepted; every tampered proof gets the verdict its bytes
call for (0: the check fails, -1: malformed); verdicts equal the oracle's `Marlin::verify`; bisection
isolates exactly the bad proofs of a batch whatever the randomiser stream."""
import json
import os
import struct

import pytest

from marlin_b200 import api, r1cs as gr1cs
from oracle import ec, kzg, marlin as omarlin
from oracle import rng as orng
from oracle import transcript as T
from oracle.params import BLS12_381, BN254

import tests_golden as golden

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCHEMES = {"marlin_kzg10": kzg.MARLIN, "sonic_kzg10": kzg.SONIC}


@pytest.fixture(scope="module")
def gctx(b2m_ctx):
    c = api.Context.__new__(api.Context)
    c.handle = b2m_ctx
    return c


def rng(seed=7):
    return api.ZkRng(bytes([seed]) * 32, 20)


class Setup:
    """GPU SRS (from the trapdoor), index and verifier key of one circuit; prove() makes GPU proofs of it."""

    def __init__(self, ctx, curve, pc, gcirc, md, beta=0x1234567, gamma=7, g=None):
        self.curve, self.pc, self.gcirc = curve, pc, gcirc
        self.m = api.Marlin(curve.name, pc, ctx=ctx)
        self.beta, self.gamma, self.g = beta, gamma, g or curve.g
        # SonicKZG10 commits to g_1 / g_2 with the gamma powers of their bounds |H| - 2 and |K| - 2: keep those of every power of two
        bounds = [(1 << k) - 2 for k in range(2, md.bit_length() + 1) if (1 << k) - 2 <= md]
        self.srs = self.m.srs_from_trapdoor(md, beta=beta, g=g, gamma=gamma, degree_bounds=bounds)
        self.pk = self.m.index(self.srs, gcirc)
        self.vk = self.m.verifier_key(self.pk, self.srs)
        self.public = gcirc.public_input()

    def prove(self, seed=0):
        return self.m.prove(self.pk, self.gcirc, api.ZkRng(bytes([seed]) * 32, 12))

    def verdicts(self, proofs, inputs=None, seed=7):
        return self.m.verify_batch(self.vk, inputs or [self.public] * len(proofs), proofs, rng(seed))

    def close(self):
        self.vk.close()
        self.pk.close()
        self.srs.close()


def dummy(ctx, curve, pc, log_n):
    f = curve.fr
    r = orng.test_rng()
    a, b = orng.field_rand(f, r), orng.field_rand(f, r)
    n = 1 << log_n
    return Setup(ctx, curve, pc, gr1cs.dummy_circuit(0 if curve is BLS12_381 else 1, a, b, 10, n), api.max_degree(n, n, 3 * n))


def layout(curve, pc, data):
    """byte offsets of the proof's parts: points (commitments, shifted commitments, W's), evaluations, random_v option bytes"""
    nq, nr = curve.fq.nbytes, curve.fr.nbytes
    off, comms, shifted, ws, rv_flags, evals = 8, [], [], [], [], []
    for _ in range(3):
        n = struct.unpack_from("<Q", data, off)[0]
        off += 8
        for _ in range(n):
            comms.append(off)
            off += nq
            if pc == "marlin_kzg10":
                has = data[off]
                off += 1
                if has:
                    shifted.append(off)
                    off += nq
    off += 8
    evals = [off + i * nr for i in range(4)]
    off += 4 * nr + 8 + 3 + 8
    for _ in range(2):
        ws.append(off)
        off += nq
        rv_flags.append(off)
        off += 1 + (nr if data[off] else 0)
    return {"comms": comms, "shifted": shifted, "ws": ws, "rv_flags": rv_flags, "evals": evals}


def put(data, off, blob):
    return data[:off] + blob + data[off + len(blob):]


def add_one_fr(curve, data, off):
    nr = curve.fr.nbytes
    v = (int.from_bytes(data[off:off + nr], "little") + 1) % curve.fr.p
    return put(data, off, v.to_bytes(nr, "little"))


def tampered(curve, pc, proof):
    """(name, bytes, expected verdict) for every tampering the check must catch"""
    L = layout(curve, pc, proof)
    other = T.g1_compressed(curve, ec.scalar_mul(curve, 5, curve.g))
    nr, nq = curve.fr.nbytes, curve.fq.nbytes
    out = []
    for i, off in enumerate(L["evals"]):
        out.append((f"eval{i}+1", add_one_fr(curve, proof, off), False))
    for kind in ("comms", "shifted", "ws"):
        for i, off in enumerate(L[kind]):
            out.append((f"{kind}{i}", put(proof, off, other), False))
    f0, f1 = L["rv_flags"]
    assert proof[f0] == 1 and proof[f1] == 0
    out.append(("random_v+1", add_one_fr(curve, proof, f0 + 1), False))
    out.append(("random_v dropped", proof[:f0] + b"\x00" + proof[f0 + 1 + nr:], False))
    out.append(("random_v added", proof[:f1] + b"\x01" + (5).to_bytes(nr, "little") + proof[f1 + 1:], False))
    both = bytearray(proof)
    both[L["comms"][0] + nq - 1] |= 0xc0
    p_bytes = bytearray(curve.fq.p.to_bytes(nq, "little"))
    out += [("truncated", proof[:-1], None), ("extended", proof + b"\x00", None), ("both flags", bytes(both), None),
            ("x >= p", put(proof, L["ws"][0], bytes(p_bytes)), None), ("eval >= r", put(proof, L["evals"][0], curve.fr.p.to_bytes(nr, "little")), None)]
    if curve is BLS12_381:  # a curve point outside the prime-order subgroup (cofactor not cleared)
        fq = curve.fq
        x = next(x for x in range(1, 1000) if pow((x ** 3 + curve.b) % fq.p, (fq.p - 1) // 2, fq.p) == 1)
        y = pow((x ** 3 + curve.b) % fq.p, (fq.p + 1) // 4, fq.p)
        out.append(("not in subgroup", put(proof, L["comms"][1], T.g1_compressed(curve, (x, y))), None))
    return out


@pytest.mark.parametrize("pc", list(SCHEMES))
@pytest.mark.parametrize("curve", [BLS12_381, BN254], ids=lambda c: c.name)
def test_accept_reject_malformed(gctx, curve, pc):
    s = dummy(gctx, curve, pc, 5)
    try:
        proof = s.prove()
        assert s.m.verify(s.vk, s.public, proof, rng())
        wrong = [(x + 1) % curve.fr.p for x in s.public]  # reference src/test.rs:158-161
        assert not s.m.verify(s.vk, wrong, proof, rng())
        cases = tampered(curve, pc, proof)
        got = s.verdicts([b for _, b, _ in cases])
        assert [(n, v) for (n, _, _), v in zip(cases, got)] == [(n, e) for n, _, e in cases]
    finally:
        s.close()


REF_SHAPES = {"tall_big": (100, 25), "tall_small": (26, 25), "squat_big": (25, 100), "squat_small": (25, 26), "square": (25, 25)}


@pytest.mark.parametrize("pc", list(SCHEMES))
@pytest.mark.parametrize("curve", [BLS12_381, BN254], ids=lambda c: c.name)
def test_reference_shapes_and_sizes(gctx, curve, pc):
    """the reference's test circuits [src/test.rs:132-203] and DummyCircuit 2^4 .. 2^12, each accepted and each rejected for a wrong
    public input, all in one batch"""
    cid = 0 if curve is BLS12_381 else 1
    f = curve.fr
    r = orng.test_rng()
    a, b = orng.field_rand(f, r), orng.field_rand(f, r)
    setups = []
    for nc, nv in REF_SHAPES.values():
        c = gr1cs.test_circuit(cid, a, b, nc, nv)
        setups.append(Setup(gctx, curve, pc, c, api.max_degree(max(nc, nv), max(nc, nv), 4 * max(nc, nv))))
    for log_n in (4, 8, 12):
        setups.append(dummy(gctx, curve, pc, log_n))
    try:
        for s in setups:
            proof = s.prove(3)
            wrong = [(x + 1) % f.p for x in s.public]
            assert s.verdicts([proof, proof], [s.public, wrong]) == [True, False]
    finally:
        for s in setups:
            s.close()


def oracle_key(s, scheme):
    """the oracle's verifier key from the same public data, on an SRS with the GPU key's max degree (lazy powers: trapdoor)"""
    curve = s.curve
    nv, nc, nnz = struct.unpack_from("<QQQ", s.pk.vk_bytes, 0)
    osrs = kzg.UniversalParams(curve, s.srs.max_degree, s.beta, s.g, s.gamma, "lazy")
    lq = s.pk.index_comms.shape[1] // 2
    comms = [tuple(curve.fq.from_mont(sum(int(p[k * lq + i]) << (64 * i) for i in range(lq))) for k in range(2)) for p in s.pk.index_comms]
    return omarlin.verifier_key_from_public(curve, scheme, osrs, nc, nv, nnz, comms)


def oracle_verdict(curve, scheme, opk, public, data, g2=None):
    try:
        proof = omarlin.deserialize_proof(curve, scheme, data)
    except Exception:
        return None
    try:
        return bool(omarlin.verify(opk, public, proof, g2))
    except Exception:
        return None


@pytest.mark.parametrize("pc", list(SCHEMES))
@pytest.mark.parametrize("curve", [BLS12_381, BN254], ids=lambda c: c.name)
def test_verdicts_equal_the_oracle(gctx, curve, pc):
    """every accept / reject case above against oracle/marlin.py::verify with the trapdoor, and a few with the G2Key pairings"""
    s = dummy(gctx, curve, pc, 4)
    try:
        opk = oracle_key(s, SCHEMES[pc])
        proof = s.prove(1)
        cases = [("ok", proof)] + [(n, b) for n, b, e in tampered(curve, pc, proof) if e is not None]
        got = s.verdicts([b for _, b in cases])
        for (name, blob), v in zip(cases, got):
            assert oracle_verdict(curve, SCHEMES[pc], opk, s.public, blob) == v, name
        g2 = kzg.G2Key(opk.ck.pp, opk.ck.enforced_degree_bounds)
        for (name, blob), v in list(zip(cases, got))[:2]:
            assert oracle_verdict(curve, SCHEMES[pc], opk, s.public, blob, g2) == v, name
    finally:
        s.close()


def test_golden_oracle_proofs(gctx):
    """tests/golden/marlin_proofs.json: proofs made by the oracle, verified against an SRS and G2 half rebuilt from the trapdoor"""
    cases = json.load(open(os.path.join(ROOT, "tests", "golden", "marlin_proofs.json")))["cases"]
    for case in cases:
        curve, a, b, _, pub = golden.case_inputs(case)
        cid = 0 if curve is BLS12_381 else 1
        gcirc = (gr1cs.test_circuit(cid, a, b, case["nc"], case["nv"]) if case["circuit"] == "test"
                 else gr1cs.dummy_circuit(cid, a, b, case["nv"], case["nc"]))
        g = ec.scalar_mul(curve, golden.G_SCALAR, curve.g)
        s = Setup(gctx, curve, case["scheme"], gcirc, case["srs_max_degree"], beta=golden.BETA, gamma=golden.GAMMA, g=g)
        try:
            proof = bytes.fromhex(case["proof_hex"])
            wrong = [(x + 1) % curve.fr.p for x in pub]
            assert s.verdicts([proof, proof], [pub, wrong]) == [True, False], case["name"]
        finally:
            s.close()


def test_replay_kit_with_its_srs_file(gctx):
    """tests/golden/replay_kit: the GPU-made proofs against the ark-serialize SRS file (G2 half read from the file)"""
    kit = os.path.join(ROOT, "tests", "golden", "replay_kit")
    meta = json.load(open(os.path.join(kit, "meta.json")))
    n = 1 << meta["log_n"]
    pub = [int(v) for v in meta["public_input"]]
    for pc in SCHEMES:
        m = api.Marlin("bls12_381", pc, ctx=gctx)
        srs = m.load_srs(os.path.join(kit, "srs.bin"))
        pk = m.index(srs, gr1cs.dummy_circuit(0, int(meta["a"]), int(meta["b"]), meta["num_variables"], n))
        vk = m.verifier_key(pk, srs)
        try:
            proof = open(os.path.join(kit, f"{pc}_proof.bin"), "rb").read()
            assert m.verify_batch(vk, [pub, [pub[0] + 1]], [proof, proof], rng()) == [True, False]
        finally:
            vk.close()
            pk.close()
            srs.close()


@pytest.mark.parametrize("pc", list(SCHEMES))
def test_batch_bisection_isolates_the_bad_proofs(gctx, pc):
    curve = BLS12_381
    s = dummy(gctx, curve, pc, 6)
    try:
        distinct = [s.prove(i) for i in range(16)]
        proofs = [distinct[i % 16] for i in range(64)]  # duplicates included
        inputs = [s.public] * 64
        assert s.verdicts(proofs, inputs) == [True] * 64
        bad = {5: "eval", 33: "w", 60: "input"}
        L = layout(curve, pc, proofs[5])
        proofs[5] = add_one_fr(curve, proofs[5], L["evals"][2])
        proofs[33] = put(proofs[33], layout(curve, pc, proofs[33])["ws"][1], T.g1_compressed(curve, ec.scalar_mul(curve, 9, curve.g)))
        inputs[60] = [(s.public[0] + 1) % curve.fr.p]
        want = [i not in bad for i in range(64)]
        for seed in (1, 2, 3):
            assert s.verdicts(proofs, inputs, seed) == want
        t = s.vk.timings()
        assert t["proofs"] == 64 and t["checks"] > 1 and t["bisection_ms"] > 0
    finally:
        s.close()


def test_missing_rng_is_an_error(gctx):
    s = dummy(gctx, BN254, "marlin_kzg10", 4)
    try:
        from marlin_b200 import _lib
        with pytest.raises(_lib.B2MError) as e:
            s.m.verify_batch(s.vk, [s.public], [s.prove()], None)
        assert e.value.code == 7
    finally:
        s.close()
