"""Random Level-1 opening sets for the `PC::check_combinations` tests, made and checked by the oracle (oracle/kzg.py): polynomials
(some hiding, some degree-bounded), arbitrary linear combinations with `LCTerm::One` terms, a query set over two points, the
evaluations and `open_combinations` proofs -- and their `api.OpeningSet` form (compressed point bytes)."""
import random

from marlin_b200 import api
from oracle import kzg
from oracle import rng as orng
from oracle import transcript as T
from oracle.poly import evaluate

D = 40                # SRS max degree
SUPPORTED = 30        # trimmed degree
BOUNDS = (12, 20)     # enforced degree bounds
HIDING = 1


def pp_for(curve, beta=0x1234567, gamma=7):
    """the oracle twin of `Marlin.srs_from_trapdoor(D, beta, gamma=gamma)`"""
    return kzg.UniversalParams(curve, D, beta, curve.g, gamma)


def ck_for(pp, scheme):
    return kzg.CommitterKey(pp, SUPPORTED, HIDING, list(BOUNDS), scheme)


class OSet:
    """One opening set in oracle form (labels -> polynomials / commitments / values) and its api.OpeningSet."""

    def __init__(self, ck, polys, comms, rands, lcs, query_set, evaluations, proofs, xi):
        self.ck, self.polys, self.comms, self.rands, self.lcs = ck, polys, comms, rands, lcs
        self.query_set, self.evaluations, self.proofs, self.xi = query_set, evaluations, proofs, xi
        self.bounds = {p.label: p.degree_bound for p in polys}

    def check(self, g2=None):
        return kzg.check_combinations(self.ck, self.lcs, {p.label: c for p, c in zip(self.polys, self.comms)}, self.bounds, self.query_set,
                                      self.evaluations, self.proofs, self.xi, g2)

    def api_set(self):
        curve = self.ck.curve
        comms = {p.label: T.g1_compressed(curve, c.comm) for p, c in zip(self.polys, self.comms)}
        shifted = {p.label: T.g1_compressed(curve, c.shifted) for p, c in zip(self.polys, self.comms) if c.shifted is not None}
        return api.OpeningSet(comms, list(self.query_set), dict(self.evaluations),
                              [(T.g1_compressed(curve, w), rv) for w, rv in self.proofs], self.xi,
                              lcs=[(lc.label, list(lc.terms)) for lc in self.lcs],
                              degree_bounds={k: v for k, v in self.bounds.items() if v is not None}, shifted=shifted)


def lc_values(ck, polys, lcs, query_set):
    """{(lc label, point): value}: the LC's polynomials at the point plus its LCTerm::One coefficients"""
    p = ck.curve.fr.p
    by = {q.label: q for q in polys}
    out = {}
    for lc_label, (_, z) in query_set:
        lc = next(x for x in lcs if x.label == lc_label)
        out[(lc_label, z)] = sum(c * (1 if t is None else evaluate(by[t].coeffs, z, p)) for c, t in lc.terms) % p
    return out


def random_set(ck, seed, n_plain=4, bounded=(12,), engine=None):
    """Polynomials a0.. (plain, every other one hiding) and b0.. (one per entry of `bounded`, that degree bound); LCs: each
    bounded polynomial alone, `mix` (two plain polynomials and a constant), `solo` (one scaled plain polynomial) and one
    identity LC per remaining plain polynomial; points "beta" and "gamma", every LC queried at one or both."""
    R = random.Random(seed)
    curve = ck.curve
    p = curve.fr.p
    polys = []
    for i in range(n_plain):
        deg = R.randrange(1, SUPPORTED + 1)
        polys.append(kzg.LabeledPoly(f"a{i}", [R.randrange(p) for _ in range(deg + 1)], None, HIDING if i % 2 else None))
    for i, d in enumerate(bounded):
        polys.append(kzg.LabeledPoly(f"b{i}", [R.randrange(p) for _ in range(R.randrange(1, d + 1))], d, HIDING if i % 2 == 0 else None))
    zr = orng.ChaChaRng(bytes([seed % 256]) * 32, rounds=12)
    engine = engine or kzg.Engine(use_trapdoor=True)
    comms, rands = kzg.commit(engine, ck, polys, zr)
    lcs = [kzg.LinearCombination(f"lc_b{i}", [(1, f"b{i}")]) for i in range(len(bounded))]
    lcs.append(kzg.LinearCombination("mix", [(R.randrange(p), "a0"), (R.randrange(p), "a1"), (R.randrange(p), None)]))
    lcs.append(kzg.LinearCombination("solo", [(R.randrange(p), "a2")]))
    lcs += [kzg.LinearCombination(f"id_a{i}", [(1, f"a{i}")]) for i in range(3, n_plain)]
    pts = {"beta": R.randrange(p), "gamma": R.randrange(p)}
    query_set = []
    for k, lc in enumerate(lcs):
        for pl in (["beta", "gamma"] if k % 3 == 0 else ["beta"] if k % 3 == 1 else ["gamma"]):
            query_set.append((lc.label, (pl, pts[pl])))
    xi = R.randrange(p)
    proofs = kzg.open_combinations(engine, ck, lcs, polys, rands, query_set, xi)
    return OSet(ck, polys, comms, rands, lcs, query_set, lc_values(ck, polys, lcs, query_set), proofs, xi)
