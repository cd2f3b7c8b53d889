"""CPU: the optimal-ate pairing of marlin_b200/csrc/pairing.cuh compiled for the host (tests/host/pairing_host_shim.cpp), on all
three curves: non-degeneracy and order r, bilinearity on GT values, "product == 1" decisions equal to the reduced Tate pairing
of pairing_host.hpp and of the oracle, GT values equal to the Python restatement in tests/pairing_ate_oracle.py, and the
prepared-line counts."""
import ctypes
import os
import random
import subprocess

import pytest

import pairing_ate_oracle as A
from oracle import ec

HERE = os.path.dirname(os.path.abspath(__file__))
IDS = {0: "bls12_381", 1: "bn254", 2: "bls12_377"}
CURVE_IDS = [0, 1, 2]


@pytest.fixture(scope="module")
def hostlib(tmp_path_factory):
    src = os.path.join(HERE, "host", "pairing_host_shim.cpp")
    so = str(tmp_path_factory.mktemp("pairing") / "libpairing_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-DB2M_HOST_LIGHT_INLINE", "-shared", "-fPIC", "-x", "c++", src, "-o", so])
    return ctypes.CDLL(so)


def nq(curve):
    return curve.fq.nbytes // 4


def g1_limbs(curve, pts):
    n = nq(curve)
    words = []
    for P in pts:
        for c in ((0, 0) if P is None else P):
            words += [(c >> (32 * i)) & 0xffffffff for i in range(n)]
    return (ctypes.c_uint32 * max(1, len(words)))(*words)


def run(lib, ci, mode, pairs):
    curve, tw = A.CURVES[ci], A.Twist(A.CURVES[ci])
    pts = g1_limbs(curve, [P for P, _ in pairs])
    g2 = b"".join(tw.uncompressed(Q) for _, Q in pairs) or b"\0"
    ok = ctypes.c_int(-1)
    out = (ctypes.c_uint32 * (12 * nq(curve)))()
    rc = lib.pairing_product(ci, mode, len(pairs), pts, g2, ctypes.byref(ok), out)
    assert rc == 0, rc
    gt = [sum(out[k * nq(curve) + i] << (32 * i) for i in range(nq(curve))) for k in range(12)]
    return ok.value, gt


def gt_value(lib, ci, pairs):
    return run(lib, ci, 1, pairs)[1]


def ate_is_one(lib, ci, pairs):
    return run(lib, ci, 0, pairs)[0] == 1


def tate_is_one(lib, ci, pairs):
    return run(lib, ci, 2, pairs)[0] == 1


def gt_pow(ci, v, k):
    return A.engine(A.CURVES[ci]).Fq12(v).pow(k).c


ONE = [1] + [0] * 11


@pytest.mark.parametrize("ci", CURVE_IDS, ids=IDS.get)
def test_line_counts_match_loop_constants(hostlib, ci):
    d = A.loop_digits(IDS[ci])
    _, _, bn = A.LOOPS[IDS[ci]]
    want = (len(d) - 1) + sum(1 for x in d[1:] if x) + (2 if bn else 0)
    assert hostlib.ate_lines_per_point(ci) == want
    assert want == {0: 68, 1: 88, 2: 69}[ci]


@pytest.mark.parametrize("ci", CURVE_IDS, ids=IDS.get)
def test_non_degenerate_order_r_and_bilinear(hostlib, ci):
    curve, tw = A.CURVES[ci], A.Twist(A.CURVES[ci])
    r = curve.fr.p
    e = gt_value(hostlib, ci, [(curve.g, tw.gen)])
    assert e != ONE
    assert gt_pow(ci, e, r) == ONE
    rnd = random.Random(100 + ci)
    a, b = rnd.randrange(1, r), rnd.randrange(1, r)
    eab = gt_value(hostlib, ci, [(ec.scalar_mul(curve, a, curve.g), tw.smul(b, tw.gen))])
    assert eab == gt_pow(ci, e, a * b % r)


@pytest.mark.parametrize("ci", CURVE_IDS, ids=IDS.get)
def test_gt_values_match_python_restatement(hostlib, ci):
    curve, tw = A.CURVES[ci], A.Twist(A.CURVES[ci])
    rnd = random.Random(200 + ci)
    P = ec.scalar_mul(curve, rnd.randrange(1, curve.fr.p), curve.g)
    Q = tw.smul(rnd.randrange(1, curve.fr.p), tw.gen)
    assert gt_value(hostlib, ci, [(P, Q)]) == A.pairing_product(curve, [(P, Q)])
    pairs = [(curve.g, tw.gen), (P, Q)]
    assert gt_value(hostlib, ci, pairs) == A.pairing_product(curve, pairs)


def random_products(ci, rnd, count):
    """seeded products that are one and not one: 1 to 6 pairs, infinity in either group, repeated G2 points, P against -P"""
    curve, tw = A.CURVES[ci], A.Twist(A.CURVES[ci])
    r = curve.fr.p
    qs = [tw.gen, tw.smul(rnd.randrange(1, r), tw.gen)]
    out = []
    for t in range(count):
        n = 1 + t % 6
        # scalars a_i, b_i with sum a_i b_i = 0 make the product one
        a = [rnd.randrange(1, r) for _ in range(n)]
        b = [rnd.randrange(1, r) for _ in range(n)]
        if n > 1:
            b[-1] = -sum(x * y for x, y in zip(a[:-1], b[:-1])) * pow(a[-1], -1, r) % r
        if t % 3 == 2 and n > 1:
            b[0] = (b[0] + 1) % r  # not one
        pairs = []
        for i in range(n):
            # e(a_i b_i G, Q0): every pair repeats the G2 point Q0
            pairs.append((ec.scalar_mul(curve, a[i] * b[i] % r, curve.g) if a[i] * b[i] % r else None, qs[0]))
        if t % 5 == 1:
            pairs.append((None, qs[1]))  # G1 at infinity
        if t % 5 == 3:
            pairs.append((ec.scalar_mul(curve, a[0], curve.g), None))  # G2 at infinity
        if t % 7 == 4:
            P = ec.scalar_mul(curve, b[0], curve.g)
            pairs += [(P, qs[1]), (ec.affine_neg(curve, P), qs[1])]  # P against -P
        out.append(pairs)
    return out


@pytest.mark.parametrize("ci", CURVE_IDS, ids=IDS.get)
def test_decisions_match_tate(hostlib, ci):
    rnd = random.Random(300 + ci)
    products = random_products(ci, rnd, 36)
    got = [ate_is_one(hostlib, ci, pr) for pr in products]
    assert got == [tate_is_one(hostlib, ci, pr) for pr in products]
    assert any(got) and not all(got)
    assert ate_is_one(hostlib, ci, [])
    # the oracle's reduced Tate pairing on a few of them
    curve, eng = A.CURVES[ci], A.engine(A.CURVES[ci])
    for pr, g in list(zip(products, got))[:4]:
        untw = [(P, None if Q is None else eng.untwist(*Q)) for P, Q in pr]
        assert eng.pairing_product_is_one([(P, Q) for P, Q in untw if P is not None and Q is not None]) == g


@pytest.mark.parametrize("ci", CURVE_IDS, ids=IDS.get)
def test_invalid_inputs_rejected(hostlib, ci):
    curve, tw = A.CURVES[ci], A.Twist(A.CURVES[ci])
    ok = ctypes.c_int()
    off = (curve.g[0], (curve.g[1] + 1) % curve.fq.p)
    assert hostlib.pairing_product(ci, 0, 1, g1_limbs(curve, [off]), tw.uncompressed(tw.gen), ctypes.byref(ok), None) == -2
    x, y = tw.gen
    bad = tw.uncompressed((x, (y[0], (y[1] + 1) % curve.fq.p)))
    assert hostlib.pairing_product(ci, 0, 1, g1_limbs(curve, [curve.g]), bad, ctypes.byref(ok), None) == -1
    big = curve.fq.p.to_bytes(curve.fq.nbytes, "little") + tw.uncompressed(tw.gen)[curve.fq.nbytes:]
    assert hostlib.pairing_product(ci, 0, 1, g1_limbs(curve, [curve.g]), big, ctypes.byref(ok), None) == -1
