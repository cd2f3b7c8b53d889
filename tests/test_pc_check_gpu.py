"""GPU: Level-1 `PC::check_combinations` / `batch_check` / `check` (b2m_pc_vk_create, b2m_pc_check_combinations) for MarlinKZG10
and SonicKZG10 on all three curves.  Honest sets -- opened by the product (b2m_ck_commit + open_combinations) and by the oracle --
are accepted; each tampering rejects exactly its set; malformed sets get -1; upstream's `Err` cases fail the call before any rng
draw; bisection isolates the bad sets and draws the rng words a node-by-node model predicts; Marlin proofs' own LCs agree with
`Marlin.verify`.  Every verdict is compared with the oracle's check_combinations (trapdoor; `G2Key` pairings for a few)."""
import ctypes
import random

import numpy as np
import pytest

import b2m_testutil as util
import bls12_377_oracle as B
import pc_check_oracle as P
from marlin_b200 import _lib, api
from oracle import ahp, ec, kzg, marlin as omarlin
from oracle import transcript as T
from oracle.params import BLS12_381, BN254
from oracle.rng import u128_rand
from test_verify_gpu import dummy, gctx, oracle_key  # noqa: F401  (gctx: fixture)

pytestmark = pytest.mark.gpu
B.register()
CURVES = {"bls12_381": BLS12_381, "bn254": BN254, "bls12_377": B.BLS12_377}
SCHEMES = {"marlin_kzg10": kzg.MARLIN, "sonic_kzg10": kzg.SONIC}
CONFIGS = [(c, pc) for c in CURVES for pc in SCHEMES]
IDS = [f"{c}-{pc}" for c, pc in CONFIGS]
BETA = 0x1234567
_ENV = {}


class Env:
    """GPU SRS from the trapdoor, its committer key and PC verifier key, and the oracle's twins"""

    def __init__(self, ctx, cname, pc):
        self.curve = CURVES[cname]
        self.cid = {"bls12_381": _lib.CURVE_BLS12_381, "bn254": _lib.CURVE_BN254, "bls12_377": _lib.CURVE_BLS12_377}[cname]
        self.pc = pc
        self.m = api.Marlin(cname, pc, ctx=ctx)
        self.srs = self.m.srs_from_trapdoor(P.D, beta=BETA, gamma=7, degree_bounds=list(P.BOUNDS))
        self.ck = self.m.trim(self.srs, P.SUPPORTED, P.HIDING, list(P.BOUNDS))
        self.vk = self.m.pc_verifier_key(self.srs, P.BOUNDS)
        self.pp = P.pp_for(self.curve, BETA)
        self.ock = P.ck_for(self.pp, SCHEMES[pc])

    def close(self):
        self.vk.close()
        self.ck.close()
        self.srs.close()


def env(ctx, cname, pc):
    if (cname, pc) not in _ENV:
        _ENV[(cname, pc)] = Env(ctx, cname, pc)
    return _ENV[(cname, pc)]


@pytest.fixture(scope="module", autouse=True)
def _close_envs():
    yield
    for e in _ENV.values():
        e.close()
    _ENV.clear()


def rng(seed=3):
    return api.ZkRng(bytes([seed]) * 32, 20)


def oracle_check(e, s, g2=None):
    """the oracle's check_combinations of an api.OpeningSet (None: a point does not decode or a value is not below r)"""
    curve, r = e.curve, e.curve.fr.p

    def pt(b):  # ark-serialize's checks: flags, x < p, the curve, the prime-order subgroup
        b = bytes(b)
        if b[-1] & 0xc0 == 0xc0:
            raise ValueError("both flags")
        q = omarlin._g1_decompress(curve, b)
        if q is not None and curve is not BN254 and ec.affine_add(curve, ec.scalar_mul(curve, r - 1, q), q) is not None:  # r q != O
            raise ValueError("not in the subgroup")
        return q
    try:
        comms = {l: kzg.Commitment(pt(c), pt(s.shifted[l]) if l in s.shifted else None) for l, c in s.commitments.items()}
        proofs = [(pt(w), rv) for w, rv in s.proofs]
    except Exception:
        return None
    if any(v >= r for v in s.evaluations.values()) or any(rv is not None and rv >= r for _, rv in s.proofs):
        return None
    lcs = [kzg.LinearCombination(l, [(c % r, t) for c, t in terms]) for l, terms in (s.lcs or [(l, [(1, l)]) for l in s.commitments])]
    bounds = {l: s.degree_bounds.get(l) for l in s.commitments}
    if SCHEMES[e.pc] == kzg.MARLIN and any(bounds[l] is not None and comms[l].shifted is None for l in comms):
        return None
    return bool(kzg.check_combinations(e.ock, lcs, comms, bounds, s.query_set, s.evaluations, proofs, s.challenge % r, g2))


def product_set(e, seed, bounded):
    """a random_set's polynomials, LCs and queries, committed and opened by the product; commitments as affine limbs"""
    o = P.random_set(e.ock, seed, bounded=bounded)
    curve, cid = e.curve, e.cid
    gp = [(util.fr_to_mont_limbs(curve, q.coeffs), q.degree_bound, q.hiding_bound) for q in o.polys]
    comm, shifted, rand, srand = e.m.commit(e.ck, gp, api.ZkRng(bytes([seed]) * 32, 12))
    label_idx = {q.label: i for i, q in enumerate(o.polys)}
    lcs = sorted(o.lcs, key=lambda lc: lc.label)
    lc_idx = {lc.label: i for i, lc in enumerate(lcs)}
    pts = {pl: z for _, (pl, z) in o.query_set}
    pls = sorted(pts)
    glcs = [[(util.fr_to_mont_limbs(curve, [c])[0], None if t is None else label_idx[t]) for c, t in lc.terms] for lc in lcs]
    gqs = [(lc_idx[l], pls.index(pl)) for l, (pl, _) in o.query_set]
    got = e.m.open_combinations(e.ck, gp, rand, srand, glcs, gqs, util.fr_to_mont_limbs(curve, [pts[pl] for pl in pls]),
                                util.fr_to_mont_limbs(curve, [o.xi])[0])
    fr = lambda a: util.fr_from_mont_limbs(curve, np.asarray(a).reshape(1, 4))[0]  # noqa: E731
    return api.OpeningSet({q.label: comm[i] for i, q in enumerate(o.polys)}, list(o.query_set), dict(o.evaluations),
                          [(w, None if rv is None else fr(rv)) for w, rv in got], o.xi, lcs=[(lc.label, list(lc.terms)) for lc in o.lcs],
                          degree_bounds={q.label: q.degree_bound for q in o.polys if q.degree_bound is not None},
                          shifted={q.label: shifted[i] for i, q in enumerate(o.polys) if q.degree_bound is not None and e.m.pc == _lib.PC_MARLIN_KZG10})


def as_bytes(e, s):
    """an api.OpeningSet with every point as compressed bytes (the oracle reads those)"""
    def b(p):
        return p if isinstance(p, (bytes, bytearray)) else api.g1_to_bytes(e.m.ctx, e.cid, p, True).tobytes()
    return api.OpeningSet({l: b(c) for l, c in s.commitments.items()}, s.query_set, dict(s.evaluations), [(b(w), rv) for w, rv in s.proofs],
                          s.challenge, lcs=s.lcs, degree_bounds=dict(s.degree_bounds), shifted={l: b(c) for l, c in s.shifted.items()})


def honest_sets(e, pc):
    bounded = [(12,), (12, 20), ()] if pc == "sonic_kzg10" else [(12,), (20,), ()]
    sets = [as_bytes(e, product_set(e, 11 + k, b)) for k, b in enumerate(bounded)]
    sets += [P.random_set(e.ock, 21 + k, bounded=b).api_set() for k, b in enumerate(bounded)]
    return sets


def copy(s):
    return api.OpeningSet(dict(s.commitments), list(s.query_set), dict(s.evaluations), list(s.proofs), s.challenge,
                          lcs=[(l, list(t)) for l, t in s.lcs], degree_bounds=dict(s.degree_bounds), shifted=dict(s.shifted))


def tamperings(e, pc):
    r = e.curve.fr.p

    def eval_plus_one(s):
        k = sorted(s.evaluations)[0]
        s.evaluations[k] = (s.evaluations[k] + 1) % r

    def other_w(s):
        s.proofs = [(s.proofs[1][0], s.proofs[0][1]), (s.proofs[0][0], s.proofs[1][1])]

    def random_v(s):
        j = next(j for j, (_, rv) in enumerate(s.proofs) if rv is not None)
        s.proofs[j] = (s.proofs[j][0], (s.proofs[j][1] + 1) % r)

    def swap_comm(s):
        s.commitments["a0"], s.commitments["a1"] = s.commitments["a1"], s.commitments["a0"]

    def swap_shifted(s):
        s.shifted["b0"] = s.commitments["b0"]

    def lc_coeff(s):
        s.lcs = [(l, [((c + 1) % r, t) for c, t in terms] if l == "mix" else terms) for l, terms in s.lcs]

    def wrong_xi(s):
        s.challenge = (s.challenge + 1) % r

    def wrong_point(s):
        z = next(z for _, (pl, z) in s.query_set if pl == "beta")
        s.query_set = [(l, (pl, (p + 1) % r if pl == "beta" else p)) for l, (pl, p) in s.query_set]
        s.evaluations = {(l, (p + 1) % r if p == z else p): v for (l, p), v in s.evaluations.items()}
    ts = [eval_plus_one, other_w, random_v, swap_comm, lc_coeff, wrong_xi, wrong_point]
    return ts + ([swap_shifted] if pc == "marlin_kzg10" else [])


@pytest.mark.parametrize("cname,pc", CONFIGS, ids=IDS)
def test_accept_and_reject(gctx, cname, pc):
    e = env(gctx, cname, pc)
    sets = honest_sets(e, pc)
    assert e.m.check_combinations(e.vk, sets, rng()) == [True] * len(sets)
    assert [oracle_check(e, s) for s in sets] == [True] * len(sets)
    t = e.vk.timings()
    assert t["sets"] == len(sets) and t["checks"] == 1 and t["products"] == 1
    for tamper in tamperings(e, pc):
        for bad in (1, 4):  # a product-made and an oracle-made set
            batch = [copy(s) for s in sets]
            tamper(batch[bad])
            want = [i != bad for i in range(len(sets))]
            assert oracle_check(e, batch[bad]) is False, tamper.__name__
            assert e.m.check_combinations(e.vk, batch, rng(5)) == want, tamper.__name__


@pytest.mark.parametrize("cname,pc", [("bn254", "marlin_kzg10"), ("bn254", "sonic_kzg10")])
def test_oracle_pairings_agree(gctx, cname, pc):
    e = env(gctx, cname, pc)
    s = P.random_set(e.ock, 31, bounded=(12, 20) if pc == "sonic_kzg10" else (12,)).api_set()
    bad = copy(s)
    bad.challenge += 1
    g2 = kzg.G2Key(e.pp, P.BOUNDS)
    assert [oracle_check(e, x, g2) for x in (s, bad)] == [True, False]
    assert e.m.check_combinations(e.vk, [s, bad], rng()) == [True, False]


def corrupt_point(curve, kind, good):
    fq = curve.fq
    nb = fq.nbytes
    if kind == "flags":
        b = bytearray(good)
        b[-1] |= 0xc0
        return bytes(b)
    if kind == "x>=p":
        return (fq.p + 1).to_bytes(nb, "little")
    for x in range(1, 1000):
        rhs = (x ** 3 + curve.b) % fq.p
        square = pow(rhs, (fq.p - 1) // 2, fq.p) == 1
        if kind == "off-curve" and not square:
            return x.to_bytes(nb, "little")
        if kind == "subgroup" and square:  # a point of the curve outside the prime-order subgroup (cofactor != 1)
            return x.to_bytes(nb, "little")
    raise AssertionError(kind)


@pytest.mark.parametrize("pc", list(SCHEMES))
def test_malformed_sets(gctx, pc):
    e = env(gctx, "bls12_381", pc)
    curve, r = e.curve, e.curve.fr.p
    sets = honest_sets(e, pc)[3:]
    cases = []
    for kind in ("flags", "x>=p", "off-curve", "subgroup"):
        s = copy(sets[1])
        s.commitments["a2"] = corrupt_point(curve, kind, s.commitments["a2"])
        cases.append(s)
        s = copy(sets[1])
        s.proofs[1] = (corrupt_point(curve, kind, s.proofs[1][0]), s.proofs[1][1])
        cases.append(s)
    s = copy(sets[1])
    s.evaluations[sorted(s.evaluations)[1]] = r
    cases.append(s)
    s = copy(sets[1])
    s.proofs[0] = (s.proofs[0][0], r + 3)
    cases.append(s)
    if pc == "marlin_kzg10":
        s = copy(sets[1])
        del s.shifted["b0"]
        cases.append(s)
    for s in cases:
        assert oracle_check(e, s) is None
        assert e.m.check_combinations(e.vk, [sets[0], s, sets[2]], rng()) == [True, None, True]


@pytest.mark.parametrize("pc", list(SCHEMES))
def test_errors_before_any_draw(gctx, pc):
    e = env(gctx, "bls12_381", pc)
    sets = honest_sets(e, pc)[3:]

    def fails(bad, what):
        g = rng(9)
        with pytest.raises(_lib.B2MError) as ei:
            e.m.check_combinations(e.vk, [sets[0], sets[1], bad], g)
        assert ei.value.code == 1 and "set 2" in str(ei.value) and what in str(ei.value), str(ei.value)
        assert g.word_pos == 0
    s = copy(sets[1])  # (the set with the bounded commitment b0)
    s.lcs = [(l, terms + [(3, "a0")] if l == "lc_b0" else terms) for l, terms in s.lcs]
    fails(s, "EquationHasDegreeBounds")
    s = copy(sets[1])
    s.degree_bounds["b0"] = 13
    fails(s, "not enforced")
    arrays = api.pc_check_arrays(e.cid, [sets[0], sets[1], sets[2]], False, None)
    arrays[16][-1] = 7  # the last query names point 7 of the last set's 2
    g = rng(9)
    verdicts = np.zeros(3, dtype=np.int32)
    rc = _lib.lib().b2m_pc_check_combinations(e.vk.handle, 3, *[_lib.ptr(a) for a in arrays], ctypes.byref(g.c), _lib.ptr(verdicts))
    assert rc == 1 and b"set 2" in _lib.lib().b2m_last_error() and g.word_pos == 0
    with pytest.raises(_lib.B2MError) as ei:
        e.m.check_combinations(e.vk, sets, None)
    assert ei.value.code == 7
    assert e.m.check_combinations(e.vk, [], rng()) == []


def words_model(points, bad):
    """ChaCha words the depth-first bisection draws: four per (set, point) of every checked node"""
    def rec(a, b):
        w = 4 * sum(points[a:b])
        if b - a > 1 and any(a <= i < b for i in bad):
            h = (b - a) // 2
            w += rec(a, a + h) + rec(a + h, b)
        return w
    return rec(0, len(points))


@pytest.mark.parametrize("m", [0, 1, 7])
@pytest.mark.parametrize("cname,pc", [("bls12_381", "marlin_kzg10"), ("bn254", "sonic_kzg10"), ("bls12_377", "marlin_kzg10")])
def test_bisection(gctx, cname, pc, m):
    e = env(gctx, cname, pc)
    two = honest_sets(e, pc)[3:]
    one = [api.OpeningSet(s.commitments, [q for q in s.query_set if q[1][0] == "beta"],
                          {k: v for k, v in s.evaluations.items() if any(k == (l, z) for l, (pl, z) in s.query_set if pl == "beta")},
                          [s.proofs[0]], s.challenge, lcs=s.lcs, degree_bounds=s.degree_bounds, shifted=s.shifted) for s in two]
    pool = two + one  # two-point and one-point sets
    n = 64
    bad = set(random.Random(100 + m).sample(range(n), m))
    sets, points = [], []
    for i in range(n):
        s = copy(pool[i % len(pool)])
        if i in bad:
            s.challenge += 1
        sets.append(s)
        points.append(len(s.proofs))
    g = rng(m + 1)
    assert e.m.check_combinations(e.vk, sets, g) == [i not in bad for i in range(n)]
    assert g.word_pos == words_model(points, bad)
    for s in (sets[i] for i in sorted(bad)[:2]):
        assert oracle_check(e, s) is False


def marlin_opening_set(opk, public_input, data):
    """`Marlin::verify`'s check_combinations inputs [reference src/lib.rs:315-433], replayed by the oracle, as an api.OpeningSet"""
    curve, scheme = opk.curve, opk.scheme
    f = curve.fr
    proof = omarlin.deserialize_proof(curve, scheme, data)
    info = opk.index.info
    from oracle.poly import Domain
    dom_x = Domain(f, len(public_input) + 1)
    public_input = list(public_input) + [0] * (max(len(public_input), dom_x.size - 1) - len(public_input))
    fs = T.FiatShamirRng(omarlin.PROTOCOL_NAME + opk.vk_bytes + b"".join(T.fe_bytes(f, x) for x in public_input))
    for k in range(3):
        fs.absorb(b"".join(omarlin.commitment_to_bytes(curve, scheme, c) for c in proof.commitments[k]))
        vs = ahp.verifier_first_round(f, info, fs) if k == 0 else ahp.verifier_second_round(vs, fs) if k == 1 else ahp.verifier_third_round(vs, fs)
    labels = ["row", "col", "a_val", "b_val", "c_val", "row_col", "w", "z_a", "z_b", "mask_poly", "t", "g_1", "h_1", "g_2", "h_2"]
    bounds = [None] * 10 + [None, vs.domain_h.size - 2, None, vs.domain_k.size - 2, None]
    comms = dict(zip(labels, opk.index_comms + proof.commitments[0] + proof.commitments[1] + proof.commitments[2]))
    query_set = ahp.verifier_query_set(vs)
    fs.absorb(b"".join(T.fe_bytes(f, x) for x in proof.evaluations))
    xi = u128_rand(fs) % f.p
    evaluations, eval_labels = {}, []
    for label, (_, point) in query_set:
        if label in ahp.LC_WITH_ZERO_EVAL:
            evaluations[(label, point)] = 0
        else:
            eval_labels.append((label, point))
    eval_labels.sort(key=lambda x: x[0])
    evaluations.update(zip(eval_labels, proof.evaluations))
    lcs = ahp.construct_linear_combinations(f, public_input, lambda l, pt: evaluations[(l, pt)], vs)
    c = lambda P_: T.g1_compressed(curve, P_)  # noqa: E731
    comm = lambda x: x.comm if isinstance(x, kzg.Commitment) else x  # noqa: E731
    return api.OpeningSet({l: c(comm(x)) for l, x in comms.items()}, list(query_set), evaluations,
                          [(c(w), rv) for w, rv in proof.pc_proof], xi, lcs=[(lc.label, list(lc.terms)) for lc in lcs],
                          degree_bounds={l: b for l, b in zip(labels, bounds) if b is not None},
                          shifted={l: c(x.shifted) for l, x in comms.items() if isinstance(x, kzg.Commitment) and x.shifted is not None})


@pytest.mark.parametrize("pc", list(SCHEMES))
def test_marlin_proofs_through_check_combinations(gctx, pc):
    s = dummy(gctx, BLS12_381, pc, 4)
    try:
        opk = oracle_key(s, SCHEMES[pc])
        nv, nc, nnz = np.frombuffer(s.pk.vk_bytes[:24], dtype=np.uint64)
        vk = s.m.pc_verifier_key(s.srs, api.index_degree_bounds(int(nc), int(nnz)))
        try:
            proofs = [s.prove(i) for i in range(2)]
            wrong = [(s.public[0] + 1) % BLS12_381.fr.p] + list(s.public[1:])
            sets = [marlin_opening_set(opk, s.public, p) for p in proofs] + [marlin_opening_set(opk, wrong, proofs[0])]
            want = s.m.verify_batch(s.vk, [s.public, s.public, wrong], proofs + [proofs[0]], rng())
            assert want == [True, True, False]
            assert s.m.check_combinations(vk, sets, rng()) == want
        finally:
            vk.close()
    finally:
        s.close()


@pytest.mark.parametrize("cname,pc", [("bls12_381", "marlin_kzg10"), ("bn254", "sonic_kzg10")])
def test_batch_check_and_check(gctx, cname, pc):
    e = env(gctx, cname, pc)
    o = P.random_set(e.ock, 41, bounded=(12,))
    s = o.api_set()
    ident = [(l, [(1, l)]) for l in s.commitments]
    # the identity LCs' evaluations: each polynomial at each point
    p = e.curve.fr.p
    from oracle.poly import evaluate
    pts = sorted({q[1] for q in s.query_set})
    polys = {q.label: q for q in o.polys}
    query = [(l, pt) for l in s.commitments for pt in pts]
    evals = {(l, z): evaluate(polys[l].coeffs, z, p) for l in s.commitments for _, z in pts}
    lc_s = api.OpeningSet(s.commitments, query, evals, [], o.xi, lcs=ident, degree_bounds=s.degree_bounds, shifted=s.shifted)
    bc = api.OpeningSet(s.commitments, query, evals, [], o.xi, degree_bounds=s.degree_bounds, shifted=s.shifted)
    lcs = [kzg.LinearCombination(l, t) for l, t in ident]
    lc_s.proofs = bc.proofs = [(T.g1_compressed(e.curve, w), rv) for w, rv in
                               kzg.open_combinations(kzg.Engine(True), e.ock, lcs, o.polys, o.rands, query, o.xi)]
    bad = copy(lc_s)
    bad.challenge += 1
    bad_bc = api.OpeningSet(bad.commitments, query, evals, bad.proofs, bad.challenge, degree_bounds=s.degree_bounds, shifted=s.shifted)
    assert e.m.check_combinations(e.vk, [lc_s, bad], rng()) == [True, False]
    assert e.m.batch_check(e.vk, [bc, bad_bc], rng()) == [True, False]
    assert oracle_check(e, lc_s) is True
    # check: one point
    one = [q for q in query if q[1] == pts[0]]
    single = api.OpeningSet(s.commitments, one, {k: v for k, v in evals.items() if k[1] == pts[0][1]},
                            [(T.g1_compressed(e.curve, w), rv) for w, rv in
                             kzg.open_combinations(kzg.Engine(True), e.ock, lcs, o.polys, o.rands, one, o.xi)], o.xi,
                            degree_bounds=s.degree_bounds, shifted=s.shifted)
    assert e.m.check(e.vk, single, rng()) is True
    single.challenge += 1
    assert e.m.check(e.vk, single, rng()) is False

