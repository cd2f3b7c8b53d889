"""GPU: `b2m_verify_multi` / `api.verify_many` -- proofs of many circuits, under several verifier keys on one or two SRSs and
both PCs, checked in one batch.  Every verdict equals the entry's `verify_batch` verdict under its own key (and the oracle's
`Marlin::verify` where it is asked); a one-key call is `verify_batch` to the rng word; bisection across keys isolates exactly
the bad proofs with the depth-first bisection's rng draws; bad arguments are refused before any rng draw."""
import ctypes
import random

import pytest

import bls12_377_oracle as B
import r1cs_random as R
from marlin_b200 import _lib, api, r1cs as gr1cs
from oracle import ec
from oracle import rng as orng
from oracle.params import BLS12_381, BN254
from test_verify_bisection_gpu import dfs_words
from test_verify_gpu import SCHEMES, Setup, add_one_fr, gctx, layout, oracle_key, oracle_verdict, tampered  # noqa: F401  (gctx: fixture)

pytestmark = pytest.mark.gpu
ERR_INVALID_ARG, ERR_MISSING_RNG = 1, 7
CURVE_ID = {"bls12_381": 0, "bn254": 1, "bls12_377": 2}
# SRS 1 is Setup's default; SRS 2 has another beta (so another beta h: a second G2 group) and another g
SRS2 = dict(beta=0x7777777, g_scalar=3)


def make(ctx, curve, pc, circ, md, srs=1, n_proofs=8):
    kw = {}
    if srs == 2:
        kw = dict(beta=SRS2["beta"], g=ec.scalar_mul(curve, SRS2["g_scalar"], curve.g))
    s = Setup(ctx, curve, pc, circ, md, **kw)
    s.proofs = [s.prove(i) for i in range(n_proofs)]
    s.bad = add_one_fr(curve, s.proofs[0], layout(curve, pc, s.proofs[0])["evals"][2])
    return s


def dummy_circ(curve, log_n):
    f = curve.fr
    r = orng.test_rng()
    a, b = orng.field_rand(f, r), orng.field_rand(f, r)
    return gr1cs.dummy_circuit(CURVE_ID[curve.name], a, b, 10, 1 << log_n)


def md_for(*circs):
    return max(api.max_degree(c.num_constraints, c.num_constraints, 3 * c.num_constraints) for c in circs)


@pytest.fixture(scope="module")
def bls(gctx):
    """BLS12-381 keys: on SRS 1 DummyCircuit 2^4 and 2^6 and a general R1CS with three public inputs under MarlinKZG10, and
    2^4 and the general R1CS again under SonicKZG10; on SRS 2 DummyCircuit 2^4 and 2^5 under both PCs"""
    g = R.small_case("x4-squat-k-below-h")
    gen = g.r1cs
    d4, d5, d6 = (dummy_circ(BLS12_381, k) for k in (4, 5, 6))
    md = max(md_for(d4, d6), api.max_degree(gen.num_constraints, gen.num_constraints, g.nnz))
    keys = {
        "d4": make(gctx, BLS12_381, "marlin_kzg10", d4, md),
        "d6": make(gctx, BLS12_381, "marlin_kzg10", d6, md),
        "gen": make(gctx, BLS12_381, "marlin_kzg10", gen, md),
        "d4s": make(gctx, BLS12_381, "sonic_kzg10", d4, md),
        "gens": make(gctx, BLS12_381, "sonic_kzg10", gen, md),
        "d4@2": make(gctx, BLS12_381, "marlin_kzg10", d4, md, srs=2),
        "d5@2": make(gctx, BLS12_381, "marlin_kzg10", d5, md, srs=2),
        "d5s@2": make(gctx, BLS12_381, "sonic_kzg10", d5, md, srs=2),
    }
    yield keys
    for s in keys.values():
        s.close()


def rng(seed=5):
    return api.ZkRng(bytes([seed]) * 32, 20)


def per_key_verdicts(entries, seed=9):
    """each entry's verdict from verify_batch under its own key (one call per key)"""
    out = [None] * len(entries)
    for s in {id(e[0]): e[0] for e in entries}.values():
        idx = [i for i, e in enumerate(entries) if e[0] is s]
        got = s.m.verify_batch(s.vk, [entries[i][1] for i in idx], [entries[i][2] for i in idx], rng(seed))
        for i, v in zip(idx, got):
            out[i] = v
    return out


def many(entries, r):
    return api.verify_many([(s.vk, pub, p) for s, pub, p in entries], r)


def test_mixed_batch_all_valid(bls):
    names = ["d4", "d6", "gen", "d4s", "d4@2"]
    entries = [(bls[k], bls[k].public, p) for k in names for p in bls[k].proofs]
    random.Random(3).shuffle(entries)
    assert many(entries, rng()) == [True] * len(entries)
    t = bls["d4"].vk.timings()
    assert t == bls["d4@2"].vk.timings()  # every key of the call holds its timings
    assert t["proofs"] == len(entries) and t["keys"] == 5 and t["g2_groups"] == 2 and t["checks"] == 1 and t["products"] == 2


def test_per_entry_verdicts_equal_verify_batch_and_the_oracle(bls):
    entries, oracle_asked = [], []
    for k in ("d4", "d6", "gen", "d4s", "d4@2"):
        s = bls[k]
        p = s.proofs[1]
        mine = [(s, s.public, p), (s, [(x + 1) % BLS12_381.fr.p for x in s.public], p), (s, s.public, b"\x03" + p[1:40])]
        mine += [(s, s.public, blob) for _, blob, _ in tampered(BLS12_381, s.pc, p)]
        oracle_asked += range(len(entries), len(entries) + 6)  # valid, wrong input, malformed and three tamperings
        entries += mine
    # valid proofs presented under another circuit's key: another size, another PC's bytes, another SRS
    cross = [("d4", "d6"), ("d6", "d4"), ("d4", "d4s"), ("d4s", "d4"), ("gen", "d4"), ("d4", "d4@2"), ("d4@2", "d4"), ("d4s", "d5s@2")]
    for key, proof_of in cross:
        entries.append((bls[key], bls[key].public, bls[proof_of].proofs[2]))
        oracle_asked.append(len(entries) - 1)
    random.Random(4).shuffle(idx := list(range(len(entries))))
    entries = [entries[i] for i in idx]
    oracle_asked = {idx.index(i) for i in oracle_asked}
    got = many(entries, rng())
    assert got == per_key_verdicts(entries)
    assert got.count(True) == 5 and False in got and None in got
    opks = {}
    for i in sorted(oracle_asked):
        s, pub, blob = entries[i]
        if id(s) not in opks:
            opks[id(s)] = oracle_key(s, SCHEMES[s.pc])
        assert oracle_verdict(BLS12_381, SCHEMES[s.pc], opks[id(s)], pub, blob) == got[i], i


@pytest.mark.parametrize("key", ["d6", "d4s"])
def test_one_key_call_is_verify_batch(bls, key):
    s = bls[key]
    n = 64
    bad = set(random.Random(7).sample(range(n), 5))
    proofs = [s.bad if i in bad else s.proofs[i % 8] for i in range(n)]
    want = [i not in bad for i in range(n)]
    a, b = rng(11), rng(11)
    assert s.m.verify_batch(s.vk, [s.public] * n, proofs, a) == want
    ta = s.vk.timings()
    assert many([(s, s.public, p) for p in proofs], b) == want
    tb = s.vk.timings()
    assert a.word_pos == b.word_pos == dfs_words(n, bad)
    assert (ta["checks"], ta["products"], ta["keys"], ta["g2_groups"]) == (tb["checks"], tb["products"], 1, 1)
    calls = []

    def counted(src):
        def nxt():
            calls.append(1)
            return src.getrandbits(64)
        return api.CallbackRng(nxt)

    assert s.m.verify_batch(s.vk, [s.public] * n, proofs, counted(random.Random(1))) == want
    n_batch = len(calls)
    calls.clear()
    assert many([(s, s.public, p) for p in proofs], counted(random.Random(1))) == want
    assert len(calls) == n_batch > 0


@pytest.mark.parametrize("m", [0, 1, 7, 64])
def test_bisection_across_keys(bls, m):
    names = list(bls)
    assert len(names) >= 8
    n = 1024
    pick = random.Random(50).choices(names, k=n)
    bad = set(random.Random(60 + m).sample(range(n), m))
    entries = [(bls[k], bls[k].public, bls[k].bad if i in bad else bls[k].proofs[i % 8]) for i, k in enumerate(pick)]
    r = api.ZkRng(bytes([m + 1]) * 32, 20)
    assert many(entries, r) == [i not in bad for i in range(n)]
    assert r.word_pos == dfs_words(n, bad)
    t = bls["d4"].vk.timings()
    assert t["proofs"] == n and t["keys"] == len(names) and t["g2_groups"] == 2 and (t["checks"] == 1) == (m == 0)


@pytest.mark.parametrize("cname", ["bn254", "bls12_377"])
def test_other_curves(gctx, cname):
    curve = BN254 if cname == "bn254" else B.BLS12_377
    d4, d5 = dummy_circ(curve, 4), dummy_circ(curve, 5)
    md = md_for(d4, d5)
    keys = [make(gctx, curve, pc, c, md, n_proofs=4) for pc in SCHEMES for c in (d4, d5)]
    try:
        entries = [(s, s.public, p) for s in keys for p in s.proofs] + [(s, s.public, s.bad) for s in keys]
        entries += [(keys[0], keys[0].public, keys[1].proofs[0]), (keys[0], keys[0].public, keys[2].proofs[0])]
        random.Random(8).shuffle(entries)
        got = many(entries, rng())
        assert got.count(True) == 4 * len(keys)
        assert got == per_key_verdicts(entries)
        assert keys[0].vk.timings()["g2_groups"] == 1
    finally:
        for s in keys:
            s.close()


def raw_multi(vks, key_of, entries, r):
    """b2m_verify_multi with explicit key handles and key_of (what verify_many cannot express)"""
    n = len(entries)
    args, verdicts, _keep = api._proof_args([vks[0].curve_id] * n, [e[0] for e in entries], [e[1] for e in entries])
    h = (ctypes.c_void_p * len(vks))(*[k.handle for k in vks])
    kof = (ctypes.c_uint32 * max(n, 1))(*key_of)
    _lib.check(_lib.lib().b2m_verify_multi(len(vks), h, n, kof, *args, ctypes.byref(r.c) if r is not None else None, verdicts))
    return [verdicts[i] for i in range(n)]


def test_errors_leave_the_rng_alone(gctx, bls):
    s = bls["d4"]
    bn = make(gctx, BN254, "marlin_kzg10", dummy_circ(BN254, 4), md_for(dummy_circ(BN254, 4)), n_proofs=1)
    ctx2 = api.Context(0)
    other = make(ctx2, BLS12_381, "marlin_kzg10", dummy_circ(BLS12_381, 4), md_for(dummy_circ(BLS12_381, 4)), n_proofs=1)
    try:
        cases = [
            ("curves", lambda r: many([(s, s.public, s.proofs[0]), (bn, bn.public, bn.proofs[0])], r), ERR_INVALID_ARG),
            ("contexts", lambda r: many([(s, s.public, s.proofs[0]), (other, other.public, other.proofs[0])], r), ERR_INVALID_ARG),
            ("key_of", lambda r: raw_multi([s.vk], [0, 1], [(s.public, s.proofs[0])] * 2, r), ERR_INVALID_ARG),
            ("no rng", lambda r: many([(s, s.public, s.proofs[0])], None), ERR_MISSING_RNG),
        ]
        for name, call, code in cases:
            r = rng()
            with pytest.raises(_lib.B2MError) as e:
                call(r)
            assert e.value.code == code, name
            assert r.word_pos == 0, name
        r = rng()
        assert api.verify_many([], r) == [] and r.word_pos == 0
        assert raw_multi([s.vk], [], [], r) == [] and r.word_pos == 0
        # the same key twice in the key list is one key
        pairs = [(s.public, s.proofs[0]), (s.public, s.proofs[1]), (s.public, s.bad)]
        assert raw_multi([s.vk, s.vk], [0, 1, 1], pairs, rng()) == [1, 1, 0]
        assert s.vk.timings()["keys"] == 1
    finally:
        bn.close()
        other.close()
        ctx2.close()
