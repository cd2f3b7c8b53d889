"""The witness MSMs of an opening.  A MarlinKZG10 shifted witness pairs with powers_of_g[D - bound ..]; when that slice overlaps
the plain witness's slice powers_of_g[0 ..) or starts just past it, its scalars are summed into the plain witness's and the point
costs one MSM; a shifted witness far from the plain slice keeps an MSM of its own.  Checked through the per-kernel spans of one
prove (MSMs and (base, scalar) pairs per proof) and through byte parity of the Level-1 open with the oracle."""
import struct

import numpy as np
import pytest

import b2m_testutil as util
from marlin_b200 import api, r1cs as gr1cs
from oracle import kzg
from oracle import rng as orng
from oracle.params import CURVES

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gctx(b2m_ctx):
    c = api.Context.__new__(api.Context)
    c.handle = b2m_ctx
    return c


def profiled(ctx, fn):
    ctx.profile(True)
    try:
        fn()
    finally:
        rep = ctx.profile_report()
        ctx.profile(False)
    return rep


def commit_pairs(scheme, H, K, X):
    """(base, scalar) pairs of the three rounds' commitments: w, z_a, z_b, mask | t, g_1, h_1 | g_2, h_2 (MarlinKZG10 commits the
    bounded g_1 and g_2 twice, plain and shifted)."""
    twice = 2 if scheme == "marlin_kzg10" else 1
    return (H + 1 - X) + 2 * (H + 1) + 3 * H + H + twice * (H - 1) + 2 * H + twice * (K - 1) + (K - 1)


@pytest.mark.parametrize("curve_name,scheme,log_n", [("bls12_381", "marlin_kzg10", 10), ("bls12_381", "marlin_kzg10", 18),
                                                     ("bn254", "marlin_kzg10", 10), ("bls12_381", "sonic_kzg10", 10)])
def test_prove_msm_count_and_pairs(gctx, curve_name, scheme, log_n):
    """bench.py's key and circuit: D = |K| - 1 = 4|H| - 1.  MarlinKZG10's shifted witness of g_1 starts 2 powers past the plain
    witness at beta ([0, 3|H| - 1) and [3|H| + 1, 4|H| - 1)), the one of g_2 lies inside the plain witness at gamma ([1, |K| - 1) in
    [0, |K| - 1)): each point is one MSM, 13 per proof and 31|H| - 6 pairs (15 and 35|H| - 10 with the shifted witnesses apart).
    SonicKZG10 has no shifted witnesses: 11 MSMs, 25|H| - 4 pairs."""
    n = 1 << log_n
    m = api.Marlin(curve_name, scheme, ctx=gctx)
    srs = m.universal_setup(n, n, 3 * n, beta=0x5eed5eed5eed5eed5eed5eed, gamma=7, degree_bounds=(n - 2, 4 * n - 2))
    circ = gr1cs.dummy_circuit(m.curve_id, 0x1234567890abcdef, 0xfedcba0987654321, 10, n)
    try:
        pk = m.index(srs, circ)
        try:
            rep = profiled(gctx, lambda: m.prove(pk, circ, api.ZkRng.test_rng()))
            nv, nc, nnz = struct.unpack_from("<QQQ", pk.vk_bytes, 0)
        finally:
            pk.close()
    finally:
        srs.close()
    H, K, X, D = n, 1 << (nnz - 1).bit_length(), circ.num_instance, srs.max_degree
    assert (H, K, X, D) == (n, 4 * n, 2, 4 * n - 1)
    if scheme == "marlin_kzg10":
        msms = 13
        pairs = commit_pairs(scheme, H, K, X) + max(3 * H - 1, D) + max(K - 1, D)  # one MSM over the union of the slices per point
        assert pairs == 31 * H - 6
    else:
        msms = 11
        pairs = commit_pairs(scheme, H, K, X) + (3 * H - 1) + (K - 1)
        assert pairs == 25 * H - 4
    assert rep["msm_accumulate_kernel"]["launches"] == msms
    assert rep["msm_sort"]["launches"] == msms
    assert rep["msm_sort"]["units"] == pairs
    assert rep["msm_reduce"]["launches"] == 4  # one batch per round's commitments, one for both opening points
    if log_n == 18:
        assert rep["msm_aff_level0"]["launches"] > 0  # the batched-affine levels are on at this size


# (length, degree bound, hiding bound) per polynomial, and the MSMs the opening takes, under a key of D = 4095.  The plain witness
# pairs with powers_of_g[0, max length - 1), the shifted witness of a bounded polynomial of length l with powers_of_g[D - bound ..
# D - bound + l - 1).
D_LEVEL1 = 4095
OPEN_CASES = {
    # [145, 344) overlaps [0, 299)
    "overlap": ([(300, None, 1), (200, 3950, None)], 1),
    # [2002, 2102) starts 2 past [0, 2000), the layout of the proof's opening at beta
    "adjacent": ([(2001, None, None), (101, 2093, None)], 1),
    # [3995, 4095) starts 3895 past [0, 100)
    "far": ([(101, None, 1), (101, 100, None)], 2),
    # [95, 394) and [495, 644) merge with [0, 499); [3095, 3594) and [4085, 4095) stay apart
    "mixed": ([(200, None, None), (300, 4000, None), (500, 1000, None), (150, 3600, None), (11, 10, None)], 3),
    # shifted randomness on a merged and on a separate shifted witness: [595, 1094) merges, [4032, 4095) does not
    "hiding": ([(1000, None, 1), (500, 3500, 1), (64, 63, 1)], 2),
    # a bounded polynomial with one coefficient has a shifted commitment but no shifted witness
    "len1": ([(50, None, None), (1, 3000, 1)], 1),
}


@pytest.mark.parametrize("case", list(OPEN_CASES))
@pytest.mark.parametrize("curve_name", ["bls12_381", "bn254"])
def test_level1_open_merged_and_separate(gctx, curve_name, case):
    import random
    curve = CURVES[curve_name]
    f = curve.fr
    spec, msms = OPEN_CASES[case]
    rnd = random.Random(f"{curve_name}/{case}")
    beta, gamma = 0xabcdef12345, 11
    osrs = kzg.UniversalParams(curve, D_LEVEL1, beta, curve.g, gamma, powers_of_g="lazy")
    bounds = sorted({b for _, b, _ in spec if b is not None})
    ck = kzg.CommitterKey(osrs, D_LEVEL1, 1, bounds, kzg.MARLIN)
    polys = [kzg.LabeledPoly(f"p{i}", [rnd.randrange(1, f.p) for _ in range(length)], bound, hb) for i, (length, bound, hb) in enumerate(spec)]
    eng = kzg.Engine(use_trapdoor=True)
    _, orands = kzg.commit(eng, ck, polys, orng.ChaChaRng(bytes(range(32)), 12))
    z, xi = rnd.randrange(f.p), rnd.randrange(1 << 128)
    ow, orv = kzg.open_at_point(eng, ck, polys, orands, z, lambda k: pow(xi, k, f.p))
    rands = np.zeros((len(polys), 4, 4), dtype=np.uint64)
    srands = np.zeros((len(polys), 4, 4), dtype=np.uint64)
    for i, r in enumerate(orands):
        if r.rand:
            rands[i, :len(r.rand)] = util.fr_to_mont_limbs(curve, r.rand)
        if r.shifted_rand:
            srands[i, :len(r.shifted_rand)] = util.fr_to_mont_limbs(curve, r.shifted_rand)
    m = api.Marlin(curve_name, "marlin_kzg10", ctx=gctx)
    srs = m.srs_from_trapdoor(D_LEVEL1, beta=beta, gamma=gamma)
    try:
        out = {}

        def run():
            out["w"], out["rv"] = m.open(srs, [(util.fr_to_mont_limbs(curve, p.coeffs), p.degree_bound, p.hiding_bound) for p in polys], rands,
                                         srands, util.fr_to_mont_limbs(curve, [z])[0], util.fr_to_mont_limbs(curve, [xi])[0],
                                         max_degree_bound=max(bounds))
        rep = profiled(gctx, run)
    finally:
        srs.close()
    assert util.points_from_limbs(curve, out["w"])[0] == ow
    assert (None if out["rv"] is None else util.fr_from_mont_limbs(curve, out["rv"])[0]) == orv
    assert rep["msm_accumulate_kernel"]["launches"] == msms
