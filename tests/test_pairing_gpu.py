"""GPU: b2m_pairing_check on all three curves -- verdicts of 10^4 seeded mixed products per curve against their construction
and, on a sample, against the host build of the same pairing (tests/host/pairing_host_shim.cpp); a call larger than one
chunk; the error paths.  b2m_verify_batch with bad proofs is in tests/test_verify_bisection_gpu.py."""
import random

import numpy as np
import pytest

import pairing_ate_oracle as A
from marlin_b200 import _lib, api
from oracle import ec
from test_pairing_host import IDS, ate_is_one, hostlib  # noqa: F401  (module fixture)

pytestmark = pytest.mark.gpu
CURVE_IDS = [0, 1, 2]


@pytest.fixture(scope="module")
def ctx():
    return api.Context(0)


def mont(curve, P):
    nq = curve.fq.nbytes // 8
    if P is None:
        return np.zeros(2 * nq, dtype=np.uint64)
    v = [curve.fq.to_mont(P[0]), curve.fq.to_mont(P[1])]
    return np.array([(c >> (64 * i)) & (2 ** 64 - 1) for c in v for i in range(nq)], dtype=np.uint64)


class Pools:
    """G1 points a_i G and G2 points b_j H with known scalars: a product's verdict is sum a_i b_j == 0 mod r"""

    def __init__(self, ci, seed):
        self.curve, tw = A.CURVES[ci], A.Twist(A.CURVES[ci])
        r = self.r = self.curve.fr.p
        rnd = random.Random(seed)
        self.b = [1] + [rnd.randrange(1, r) for _ in range(3)]
        self.g2 = [tw.gen] + [tw.smul(b, tw.gen) for b in self.b[1:]] + [None]
        self.g2_bytes = [tw.uncompressed(Q) for Q in self.g2]
        self.a = [rnd.randrange(1, r) for _ in range(12)]
        self.a += [r - x for x in self.a]  # negatives
        # a point whose pairing with H cancels a[0] against b[1]: c = -a0 b1
        self.a.append(-self.a[0] * self.b[1] % r)
        self.g1 = [ec.scalar_mul(self.curve, x, self.curve.g) for x in self.a] + [None]
        self.g1m = [mont(self.curve, P) for P in self.g1]

    def product(self, rnd):
        """(pairs as (g1 pool index, g2 pool index), expected verdict)"""
        n_pos = len(self.a) - 1  # the cancelling point is the last scalar
        pairs = []
        for _ in range(rnd.randrange(0, 3)):
            i, j = rnd.randrange(12), rnd.randrange(4)
            pairs += [(i, j), (i + 12, j)]  # P against -P
        kind = rnd.randrange(5)
        if kind == 0:
            pairs += [(0, 1), (n_pos, 0)]  # e(a0 G, b1 H) e(-a0 b1 G, H)
        elif kind == 1:
            pairs.append((rnd.randrange(n_pos + 1), rnd.randrange(4)))  # not one
        elif kind == 2:
            pairs += [(len(self.g1) - 1, rnd.randrange(4)), (rnd.randrange(n_pos + 1), 4)]  # infinity in either group
        rnd.shuffle(pairs)
        s = sum(self.a[i] * self.b[j] for i, j in pairs if i < len(self.a) and j < 4) % self.r
        return pairs, s == 0


def run(ctx, ci, pools, products):
    prods = [[(pools.g1m[i], j) for i, j in pr] for pr, _ in products]
    return api.pairing_check(ctx, ci, pools.g2_bytes, prods)


@pytest.mark.parametrize("ci", CURVE_IDS, ids=IDS.get)
def test_pairing_check_matches_construction_and_host(ctx, hostlib, ci):  # noqa: F811
    pools = Pools(ci, 500 + ci)
    rnd = random.Random(600 + ci)
    products = [pools.product(rnd) for _ in range(10000)]
    got = run(ctx, ci, pools, products)
    assert got == [v for _, v in products]
    assert 0 < sum(got) < len(got)
    for k in range(0, 10000, 400):  # the host build of the same code on a sample
        pairs = [(pools.g1[i], pools.g2[j]) for i, j in products[k][0]]
        assert ate_is_one(hostlib, ci, pairs) == got[k]


def test_pairing_check_larger_than_one_chunk(ctx):
    ci = 1
    pools = Pools(ci, 700)
    rnd = random.Random(701)
    base = [pools.product(rnd) for _ in range(64)]
    products = [base[k % 64] for k in range((1 << 16) + 77)]
    assert run(ctx, ci, pools, products) == [v for _, v in products]


@pytest.mark.parametrize("ci", CURVE_IDS, ids=IDS.get)
def test_pairing_check_errors(ctx, ci):
    pools = Pools(ci, 800 + ci)
    curve = pools.curve
    assert api.pairing_check(ctx, ci, pools.g2_bytes, []) == []
    assert api.pairing_check(ctx, ci, pools.g2_bytes, [[]]) == [True]
    off = mont(curve, (curve.g[0], (curve.g[1] + 1) % curve.fq.p))
    with pytest.raises(_lib.B2MError) as e:
        api.pairing_check(ctx, ci, pools.g2_bytes, [[(pools.g1m[0], 0)], [(pools.g1m[1], 0), (off, 1)]])
    assert e.value.code == 1 and "G1 point 2" in str(e.value)
    nb = curve.fq.nbytes
    bad = bytearray(pools.g2_bytes[1])
    bad[:nb] = curve.fq.p.to_bytes(nb, "little")
    with pytest.raises(_lib.B2MError) as e:
        api.pairing_check(ctx, ci, [pools.g2_bytes[0], bytes(bad)], [[(pools.g1m[0], 0)]])
    assert e.value.code == 11 and "G2 point 1" in str(e.value)
    with pytest.raises(_lib.B2MError):
        api.pairing_check(ctx, ci, pools.g2_bytes[:1], [[(pools.g1m[0], 3)]])
