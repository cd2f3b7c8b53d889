"""Independent Python model of arkworks SRS files for the ark-SRS tests: G2 point compression / decompression on the twist
and a writer for a full-shape `KZG10::setup(D)` output (D + 1 powers_of_g, D + 2 powers_of_gamma_g, h, beta_h and, for
SonicKZG10, D + 1 neg_powers_of_h) [U ark-poly-commit 0.3 kzg10::setup, ark-serialize 0.3].  Plain integers over oracle/;
the product never imports it."""
import struct

from oracle import ec, pairing as opairing
from oracle import transcript as T
from oracle.params import BLS12_381, BN254

# standard G2 generators (x.c0, x.c1, y.c0, y.c1) [U ark-bls12-381 / ark-bn254 0.3 g2 parameters]
G2_GEN = {
    "bls12_381": (0x024aa2b2f08f0a91260805272dc51051c6e47ad4fa403b02b4510b647ae3d1770bac0326a805bbefd48056c8c121bdb8,
                  0x13e02b6052719f607dacd3a088274f65596bd0d09920b61ab5da61bbdc7f5049334cf11213945d57e5ac7d055d042b7e,
                  0x0ce5d527727d6e118cc9cdc6da2e351aadfd9baa8cbdd3a76d429a695160d12c923ac9cc3baca289e193548608b82801,
                  0x0606c4a02ea734cc32acd2b02bc28b99cb3e287e85a763af267492ab572e99ab3f370d275cec1da1aaa9075ff05f79be),
    "bn254": (0x1800deef121f1e76426a00665e5c4479674322d4f75edadd46debd5cd992f6ed,
              0x198e9393920d483a7260bfb731fb5d25f1aa493335a9e71297e485b7aef312c2,
              0x12c85ea5db8c6deb4aab71808dcb408fe3d1e7690c43d37b4ce6cc0166fa7daa,
              0x090689d0585ff075ec9e99ad690c3395bc4b313370b38ef355acdadcd122975b),
}


class G2:
    """E'(Fq2): y^2 = x^3 + b', affine points ((x0, x1), (y0, y1)), None = infinity."""

    def __init__(self, curve):
        self.curve, self.p = curve, curve.fq.p
        self.eng = opairing.for_curve(curve)
        p = self.p
        self.b = (4, 4) if curve is BLS12_381 else self.eng._fq2_mul((3, 0), self.eng._fq2_inv((9, 1)))
        g = G2_GEN[curve.name]
        self.gen = ((g[0], g[1]), (g[2], g[3]))
        assert self.on_curve(self.gen)
        self.add_ = lambda a, b: ((a[0] + b[0]) % p, (a[1] + b[1]) % p)
        self.sub_ = lambda a, b: ((a[0] - b[0]) % p, (a[1] - b[1]) % p)

    def mul_(self, a, b):
        return self.eng._fq2_mul(a, b)

    def rhs(self, x):
        x3 = self.mul_(self.mul_(x, x), x)
        return ((x3[0] + self.b[0]) % self.p, (x3[1] + self.b[1]) % self.p)

    def on_curve(self, P):
        return P is None or self.mul_(P[1], P[1]) == self.rhs(P[0])

    def add(self, P, Q):
        if P is None:
            return Q
        if Q is None:
            return P
        if P[0] == Q[0]:
            if (P[1][0] + Q[1][0]) % self.p == 0 and (P[1][1] + Q[1][1]) % self.p == 0:
                return None
            x2 = self.mul_(P[0], P[0])
            lam = self.mul_(((3 * x2[0]) % self.p, (3 * x2[1]) % self.p), self.eng._fq2_inv(((2 * P[1][0]) % self.p, (2 * P[1][1]) % self.p)))
        else:
            lam = self.mul_(self.sub_(Q[1], P[1]), self.eng._fq2_inv(self.sub_(Q[0], P[0])))
        x3 = self.sub_(self.sub_(self.mul_(lam, lam), P[0]), Q[0])
        return (x3, self.sub_(self.mul_(lam, self.sub_(P[0], x3)), P[1]))

    def smul(self, k, P):
        R = None
        while k:
            if k & 1:
                R = self.add(R, P)
            P = self.add(P, P)
            k >>= 1
        return R

    def neg(self, P):
        return None if P is None else (P[0], ((-P[1][0]) % self.p, (-P[1][1]) % self.p))

    def larger(self, y):
        """y > -y in QuadExtField's ordering (c1 first, then c0)"""
        p = self.p
        return y[1] > (p - y[1]) % p if y[1] else y[0] > (p - y[0]) % p

    def raw_point(self, start=0):
        """a twist point with x = (k, 1), cofactor not cleared"""
        k = start
        while True:
            y = self.eng._fq2_sqrt(self.rhs((k, 1)))
            if y is not None:
                return ((k, 1), y)
            k += 1

    def uncompressed(self, P):
        nb = self.curve.fq.nbytes
        if P is None:
            b = bytearray(4 * nb)
            b[-1] |= 0x40
            return bytes(b)
        return b"".join(v.to_bytes(nb, "little") for v in (P[0][0], P[0][1], P[1][0], P[1][1]))

    def compressed(self, P):
        nb = self.curve.fq.nbytes
        if P is None:
            b = bytearray(2 * nb)
            b[-1] |= 0x40
            return bytes(b)
        b = bytearray(P[0][0].to_bytes(nb, "little") + P[0][1].to_bytes(nb, "little"))
        if self.larger(P[1]):
            b[-1] |= 0x80
        return bytes(b)

    def decompress(self, blob):
        """compressed bytes -> point (no subgroup check); ValueError on bad flags / x >= p / no square root"""
        nb, p = self.curve.fq.nbytes, self.p
        x0 = int.from_bytes(blob[:nb], "little")
        x1 = int.from_bytes(blob[nb:2 * nb], "little")
        flags = x1 >> (8 * nb - 2)
        x1 &= (1 << (8 * nb - 2)) - 1
        if flags == 3 or x0 >= p or x1 >= p:
            raise ValueError("bad flags or x >= p")
        if flags == 1:
            return None
        y = self.eng._fq2_sqrt(self.rhs((x0, x1)))
        if y is None:
            raise ValueError("not on the curve")
        if self.larger(y) != (flags == 2):
            y = ((-y[0]) % p, (-y[1]) % p)
        return ((x0, x1), y)


def g1_uncompressed(curve, P):
    nb = curve.fq.nbytes
    if P is None:
        b = bytearray(2 * nb)
        b[-1] |= 0x40
        return bytes(b)
    return P[0].to_bytes(nb, "little") + P[1].to_bytes(nb, "little")


def g1_bytes(curve, P, compressed):
    return T.g1_compressed(curve, P) if compressed else g1_uncompressed(curve, P)


def kzg10_setup(curve, D, beta, gamma, sonic, compressed):
    """-> (file bytes, points) of a full-shape `KZG10::setup(D)` with trapdoor (beta, gamma) and the standard generators;
    points = dict(powers [D + 1], gamma {0..=D+1}, h, beta_h, neg {0..=D} for SonicKZG10 else {})"""
    r = curve.fr.p
    g2 = G2(curve)
    powers = [ec.scalar_mul(curve, pow(beta, i, r), curve.g) for i in range(D + 1)]
    gamma_g = ec.scalar_mul(curve, gamma, curve.g)
    gam = {i: ec.scalar_mul(curve, pow(beta, i, r), gamma_g) for i in range(D + 2)}
    h, beta_h = g2.gen, g2.smul(beta, g2.gen)
    binv = pow(beta, -1, r)
    neg = {i: g2.smul(pow(binv, i, r), g2.gen) for i in range(D + 1)} if sonic else {}
    g2b = g2.compressed if compressed else g2.uncompressed
    out = [struct.pack("<Q", len(powers))] + [g1_bytes(curve, P, compressed) for P in powers]
    out.append(struct.pack("<Q", len(gam)))
    for k in sorted(gam):
        out += [struct.pack("<Q", k), g1_bytes(curve, gam[k], compressed)]
    out += [g2b(h), g2b(beta_h), struct.pack("<Q", len(neg))]
    for k in sorted(neg):
        out += [struct.pack("<Q", k), g2b(neg[k])]
    return b"".join(out), {"powers": powers, "gamma": gam, "h": h, "beta_h": beta_h, "neg": neg}


CURVES = {"bls12_381": BLS12_381, "bn254": BN254}
