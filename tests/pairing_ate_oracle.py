"""A Python restatement of the optimal-ate pairing of marlin_b200/csrc/pairing.cuh, for tests only.

Everything runs in the oracle's single-extension Fq12 (oracle/pairing.py) on untwisted G2 points: the Miller loop takes lines
through multiples of psi(Q), evaluated at P (numerators only: the denominators lie in proper subfields, which the final
exponentiation maps to 1), BN254's extra points are pi(psi(Q)) = (x^p, y^p) and -pi^2(psi(Q)), and the final exponentiation is
one power by e (p^12 - 1) / r with the e that pairing.cuh documents: 3 for BLS12 curves, 2u (6u^2 + 3u + 1) for BN254.  So it
shares no formula with the device code beyond the loop scalar and e."""
import ark_srs_oracle
import bls12_377_oracle as B
from oracle import pairing as opairing
from oracle.params import BLS12_381, BN254

BN_U = 0x44e992b44a6909f1
# (|x| or 6u + 2 as NAF digits, most significant first), x < 0, BN
LOOPS = {
    "bls12_381": (0xd201000000010000, True, False),
    "bls12_377": (0x8508c00000000001, False, False),
    "bn254": (6 * BN_U + 2, False, True),
}
E_MULT = {"bls12_381": 3, "bls12_377": 3, "bn254": 2 * BN_U * (6 * BN_U * BN_U + 3 * BN_U + 1)}


def naf(k):
    d = []
    while k:
        z = (2 - k % 4) if k & 1 else 0
        d.append(z)
        k = (k - z) // 2
    return d[::-1]


def loop_digits(name):
    k, _, bn = LOOPS[name]
    return naf(k) if bn else [int(c) for c in bin(k)[2:]]


def engine(curve):
    if curve.name == "bls12_377":
        return B.register()
    return opairing.for_curve(curve)


class Twist:
    """E'(Fq2) points ((x0, x1), (y0, y1)) of one curve and their ark-serialize uncompressed bytes"""

    def __init__(self, curve):
        self.curve = curve
        if curve.name == "bls12_377":
            g = B.G2_GENERATOR
            self.gen = ((g[0], g[1]), (g[2], g[3]))
            self.add, self.smul = B.g2_add, lambda k, P: B.g2_mul(k, P)
            self._srs = None
        else:
            self._srs = ark_srs_oracle.G2(curve)
            self.gen = self._srs.gen
            self.add, self.smul = self._srs.add, self._srs.smul

    def neg(self, P):
        p = self.curve.fq.p
        return None if P is None else (P[0], ((-P[1][0]) % p, (-P[1][1]) % p))

    def uncompressed(self, P):
        nb = self.curve.fq.nbytes
        if P is None:
            b = bytearray(4 * nb)
            b[-1] |= 0x40
            return bytes(b)
        return b"".join(v.to_bytes(nb, "little") for v in (P[0][0], P[0][1], P[1][0], P[1][1]))


def miller_loop(curve, P, Q):
    """f for one pair: P affine G1 ints, Q a twist point"""
    eng = engine(curve)
    F = eng.Fq12
    if P is None or Q is None:
        return F.one()
    p = curve.fq.p
    xp, yp = F.from_fq(P[0]), F.from_fq(P[1])
    Qe = eng.untwist(*Q)

    def line(T, S):
        (xt, yt), (xs, ys) = T, S
        if xt == xs and yt == ys:
            return yt.scale(2) * (yp - yt) - xt.square().scale(3) * (xp - xt)
        if xt == xs:
            return xp - xt
        return (xs - xt) * (yp - yt) - (ys - yt) * (xp - xt)

    digits = loop_digits(curve.name)
    _, x_neg, bn = LOOPS[curve.name]
    f, T = F.one(), Qe
    negQ = eng.e12_neg(Qe)
    for d in digits[1:]:
        f = f.square() * line(T, T)
        T = eng.e12_add(T, T)
        if d:
            S = Qe if d == 1 else negQ
            f = f * line(T, S)
            T = eng.e12_add(T, S)
    if x_neg:  # conjugation w -> -w
        f = F([c if i % 2 == 0 else -c for i, c in enumerate(f.c)])
    if bn:
        q1 = (Qe[0].pow(p), Qe[1].pow(p))
        q2 = (Qe[0].pow(p * p), -(Qe[1].pow(p * p)))
        f = f * line(T, q1)
        T = eng.e12_add(T, q1)
        f = f * line(T, q2)
    return f


def final_exponent(curve):
    p, r = curve.fq.p, curve.fr.p
    return E_MULT[curve.name] * ((p ** 12 - 1) // r)


def pairing_product(curve, pairs):
    """prod e(P_i, Q_i) in GT: 12 ints, the coefficients of 1, w, ..., w^11"""
    F = engine(curve).Fq12
    f = F.one()
    for P, Q in pairs:
        f = f * miller_loop(curve, P, Q)
    return f.pow(final_exponent(curve)).c


CURVES = {0: BLS12_381, 1: BN254, 2: B.BLS12_377}
