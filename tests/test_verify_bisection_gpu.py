"""GPU: `b2m_verify_batch` with bad proofs at seeded positions -- batches of 64 and 1024 proofs with m in {0, 1, 7, 64}
tampered proofs, on both PCs of BLS12-381 and BN254 and MarlinKZG10 on BLS12-377.  Verdicts equal the oracle's per-proof
`Marlin::verify`, and the caller's rng ends where the depth-first bisection leaves it: the checks run level by level, but
they are the same checks, each drawing two 128-bit randomisers (8 ChaCha words) per proof."""
import random

import pytest

import bls12_377_oracle as B
from marlin_b200 import _lib, api, r1cs as gr1cs
from oracle import rng as orng
from oracle.params import BLS12_381, BN254
from test_verify_gpu import SCHEMES, Setup, add_one_fr, dummy, gctx, layout, oracle_key, oracle_verdict  # noqa: F401  (gctx: fixture)

pytestmark = pytest.mark.gpu
CONFIGS = [("bls12_381", "marlin_kzg10"), ("bls12_381", "sonic_kzg10"), ("bn254", "marlin_kzg10"), ("bn254", "sonic_kzg10"),
           ("bls12_377", "marlin_kzg10")]
WORDS_PER_PROOF = 8  # two opening points, one 128-bit randomiser (two u64, four 32-bit words) each
_SETUPS = {}


def setup_for(ctx, cname, pc):
    key = (cname, pc)
    if key not in _SETUPS:
        if cname == "bls12_377":
            B.register()
            f = B.BLS12_377.fr
            r = orng.test_rng()
            a, b = orng.field_rand(f, r), orng.field_rand(f, r)
            n = 16
            s = Setup(ctx, B.BLS12_377, pc, gr1cs.dummy_circuit(_lib.CURVE_BLS12_377, a, b, 10, n), api.max_degree(n, n, 3 * n))
        else:
            s = dummy(ctx, BLS12_381 if cname == "bls12_381" else BN254, pc, 4)
        s.distinct = [s.prove(i) for i in range(16)]
        L = layout(s.curve, pc, s.distinct[0])
        s.bad = [add_one_fr(s.curve, p, L["evals"][2]) for p in s.distinct]
        opk = oracle_key(s, SCHEMES[pc])
        s.want = {blob: oracle_verdict(s.curve, SCHEMES[pc], opk, s.public, blob) for blob in s.distinct + s.bad}
        _SETUPS[key] = s
    return _SETUPS[key]


@pytest.fixture(scope="module", autouse=True)
def _close_setups():
    yield
    for s in _SETUPS.values():
        s.close()
    _SETUPS.clear()


def dfs_words(n, bad):
    """ChaCha words the depth-first bisection draws over proofs [0, n) with the given bad set"""
    def rec(a, b):
        words = WORDS_PER_PROOF * (b - a)
        if b - a > 1 and any(a <= i < b for i in bad):
            h = (b - a) // 2
            words += rec(a, a + h) + rec(a + h, b)
        return words
    return rec(0, n)


@pytest.mark.parametrize("m", [0, 1, 7, 64])
@pytest.mark.parametrize("n", [64, 1024])
@pytest.mark.parametrize("cname,pc", CONFIGS, ids=[f"{c}-{p}" for c, p in CONFIGS])
def test_verify_batch_bad_proofs(gctx, cname, pc, n, m):
    s = setup_for(gctx, cname, pc)
    bad = set(random.Random(1000 * n + m).sample(range(n), m))
    proofs = [s.bad[i % 16] if i in bad else s.distinct[i % 16] for i in range(n)]
    want = [s.want[p] for p in proofs]
    assert want == [i not in bad for i in range(n)]  # the oracle rejects exactly the tampered proofs
    rng = api.ZkRng(bytes([m + 1]) * 32, 20)
    assert s.m.verify_batch(s.vk, [s.public] * n, proofs, rng) == want
    assert rng.word_pos == dfs_words(n, bad)
    t = s.vk.timings()
    assert t["proofs"] == n and (t["checks"] == 1) == (m == 0)
