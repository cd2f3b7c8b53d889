"""BLS12-377 for the Python oracle: its field and curve parameters, derived from the curve parameter u, and a reduced Tate
pairing over Fq12 = Fq[w] / (w^12 + 5).

The oracle package is written against `oracle.params.CurveParams`; everything but the pairing and the square root behind
compressed G1 points (p = 3 mod 4 there) is already generic over the curve.  Importing this module registers BLS12-377 with
the oracle at run time (`oracle.params.CURVES`, the pairing engine cache of `oracle.pairing.for_curve`, a G1 decompression
for q = 1 mod 4 behind `oracle.marlin.deserialize_proof`, and `b2m_testutil.CURVE_ID`), so the tests can run the oracle's
prover, KZG checks, proof deserializer and pairing verifier on the new curve.

Constants (every one re-derived and asserted here):
- u = 0x8508c00000000001, r = u^4 - u^2 + 1 (253 bits, 2-adicity 47), q = (u - 1)^2 r / 3 + u (377 bits, 2-adicity 46).
- Fr generator 22 (ark-bls12-377's; it fixes the coset-NTT shift).  Fq generator 15 (only Tonelli-Shanks needs a non-residue).
- G1: y^2 = x^3 + 1, cofactor (u - 1)^2 / 3.  Fq2 = Fq[u] / (u^2 + 5), xi = u, D-type twist y^2 = x^3 + 1 / u.
"""
import b2m_testutil
from marlin_b200 import _lib
from oracle import marlin as omarlin
from oracle import pairing as opairing
from oracle import params as oparams

U = 0x8508c00000000001
R_MOD = U ** 4 - U ** 2 + 1
Q_MOD = (U - 1) ** 2 * R_MOD // 3 + U
assert (U - 1) ** 2 * R_MOD % 3 == 0
assert R_MOD == 0x12ab655e9a2ca55660b44d1e5c37b00159aa76fed00000010a11800000000001
assert Q_MOD == 0x01ae3a4617c510eac63b05c06ca1493b1a22d9f300f5138f1ef3622fba094800170b5d44300000008508c00000000001

FR = oparams.FieldParams("bls12_377_fr", R_MOD, 22, 3)
FQ = oparams.FieldParams("bls12_377_fq", Q_MOD, 15, 7)
assert (FR.bits, FR.two_adicity, FQ.bits, FQ.two_adicity) == (253, 47, 377, 46)
assert pow(22, (R_MOD - 1) // 2, R_MOD) == R_MOD - 1 and pow(15, (Q_MOD - 1) // 2, Q_MOD) == Q_MOD - 1

G1_COFACTOR = (U - 1) ** 2 // 3
assert (Q_MOD + 1 - (U + 1)) == G1_COFACTOR * R_MOD  # #E(Fq) = q + 1 - t, trace t = u + 1
BLS12_377 = oparams.CurveParams(
    "bls12_377", FQ, FR, 1,
    0x008848defe740a67c8fc6225bf87ff5485951e2caa9d41bb188282c8bd37cb5cd5481512ffcd394eeab9b16eb21be9ef,
    0x01914a69c5102eff1f674f5d30afeec4bd7fb348ca3e52d96d182ad44fb82305c2fe3d3634a9591afd82de55559c8ea6)

BETA = 5  # u^2 = -5
assert pow(Q_MOD - BETA, (Q_MOD - 1) // 2, Q_MOD) == Q_MOD - 1, "-5 must be a non-residue"
OMEGA = pow(2, (Q_MOD - 1) // 3, Q_MOD)  # phi(x, y) = (omega x, y) acts on G1 as -u^2
# b' = 1 / u = -u / 5 on the twist, as (c0, c1)
B_TWIST = (0, (-pow(5, -1, Q_MOD)) % Q_MOD)
# ark-bls12-377's G2 generator (x.c0, x.c1, y.c0, y.c1), checked on the twist and of order r below
G2_GENERATOR = (
    0x018480be71c785fec89630a2a3841d01c565f071203e50317ea501f557db6b9b71889f52bb53540274e3e48f7c005196,
    0x00ea6040e700403170dc5a51b1b140d5532777ee6651cecbe7223ece0799c9de5cf89984bff76fe6b26bfefa6ea16afe,
    0x00690d665d446f7bd960736bcbb2efb4de03ed7274b49a58e458c282f832d204f2cf88886d8c7c2ef094094409fd4ddf,
    0x00f8169fd28355189e549da3151a70aa61ef11ac3d591bf12463b01acee304c24279b83f5e52270bd9a1cdd185eb8f93)


def fq2_mul(a, b):
    p = Q_MOD
    return ((a[0] * b[0] - BETA * a[1] * b[1]) % p, (a[0] * b[1] + a[1] * b[0]) % p)


def fq2_add(a, b):
    return ((a[0] + b[0]) % Q_MOD, (a[1] + b[1]) % Q_MOD)


def fq2_sub(a, b):
    return ((a[0] - b[0]) % Q_MOD, (a[1] - b[1]) % Q_MOD)


def fq2_inv(a):
    n = pow(a[0] * a[0] + BETA * a[1] * a[1], -1, Q_MOD)
    return (a[0] * n % Q_MOD, -a[1] * n % Q_MOD)


def fq_sqrt(a, p=Q_MOD):
    """Tonelli-Shanks (Python model of the device's); None for a non-square"""
    a %= p
    if a == 0:
        return 0
    if pow(a, (p - 1) // 2, p) != 1:
        return None
    s, t = 0, p - 1
    while t % 2 == 0:
        s, t = s + 1, t // 2
    z = next(g for g in range(2, 1000) if pow(g, (p - 1) // 2, p) == p - 1)
    m, c, x, b = s, pow(z, t, p), pow(a, (t + 1) // 2, p), pow(a, t, p)
    while b != 1:
        k, b2 = 0, b
        while b2 != 1:
            b2, k = b2 * b2 % p, k + 1
        w = pow(c, 1 << (m - k - 1), p)
        x, c = x * w % p, w * w % p
        b, m = b * c % p, k
    return x


def fq2_sqrt(a):
    """some square root of a in Fq2, None if a is not a square"""
    a0, a1 = a[0] % Q_MOD, a[1] % Q_MOD
    if a1 == 0:
        s = fq_sqrt(a0)
        if s is not None:
            return (s, 0)
        s = fq_sqrt(-a0 * pow(BETA, -1, Q_MOD))
        return None if s is None else (0, s)
    n = fq_sqrt(a0 * a0 + BETA * a1 * a1)
    if n is None:
        return None
    for sign in (1, -1):
        x = fq_sqrt((a0 + sign * n) * pow(2, -1, Q_MOD))
        if x:
            y = a1 * pow(2 * x, -1, Q_MOD) % Q_MOD
            if fq2_mul((x, y), (x, y)) == (a0, a1):
                return (x, y)
    return None


def g2_on_twist(x, y):
    return fq2_mul(y, y) == fq2_add(fq2_mul(fq2_mul(x, x), x), B_TWIST)


def g2_add(P, Q):
    if P is None:
        return Q
    if Q is None:
        return P
    (x1, y1), (x2, y2) = P, Q
    if x1 == x2:
        if fq2_add(y1, y2) == (0, 0):
            return None
        lam = fq2_mul(fq2_mul((3, 0), fq2_mul(x1, x1)), fq2_inv(fq2_mul((2, 0), y1)))
    else:
        lam = fq2_mul(fq2_sub(y2, y1), fq2_inv(fq2_sub(x2, x1)))
    x3 = fq2_sub(fq2_sub(fq2_mul(lam, lam), x1), x2)
    return (x3, fq2_sub(fq2_mul(lam, fq2_sub(x1, x3)), y1))


def g2_mul(k, P):
    acc = None
    while k:
        if k & 1:
            acc = g2_add(acc, P)
        P, k = g2_add(P, P), k >> 1
    return acc


class Bls377PairingEngine(opairing.PairingEngine):
    """The oracle's reduced Tate pairing with Fq12 = Fq[w] / (w^12 - 2 alpha w^6 + alpha^2 + beta), alpha = 0, beta = 5:
    w^6 = xi = u, D-type untwist (x, y) -> (x w^2, y w^3)."""

    def __init__(self):
        super().__init__(BLS12_377, 0, "D", None)
        self.c6, self.c0 = 0, BETA  # w^12 = -5; nothing in the base constructor reduced by c0 for alpha = 0 and a D-type twist
        x, y = (G2_GENERATOR[0], G2_GENERATOR[1]), (G2_GENERATOR[2], G2_GENERATOR[3])
        self._g2 = self.untwist(x, y)
        assert self.e12_on_curve(self._g2)

    def _fq2_mul(self, a, b):
        return fq2_mul(a, b)

    def _fq2_inv(self, a):
        return fq2_inv(a)

    def _fq2_sqrt(self, a):
        return fq2_sqrt(a)


def g1_decompress(curve, data):
    """ark-serialize compressed G1 (x little-endian, bit 7 = y is the larger root, bit 6 = infinity) with a Tonelli-Shanks
    square root; the oracle's own decoder, which takes p = 3 mod 4, serves the other curves"""
    if curve.fq.p % 4 == 3:
        return _ORACLE_G1_DECOMPRESS(curve, data)
    b = bytearray(data)
    flags = b[-1] & 0xc0
    b[-1] &= 0x3f
    if flags & 0x40:
        return None
    p = curve.fq.p
    x = int.from_bytes(bytes(b), "little")
    y = fq_sqrt(x * x * x + curve.b, p)
    if y is None:
        raise ValueError("compressed point is not on the curve")
    if bool(flags & 0x80) != (y > (p - y) % p):
        y = (p - y) % p
    return (x, y)


_ORACLE_G1_DECOMPRESS = getattr(omarlin._g1_decompress, "__wrapped__", omarlin._g1_decompress)  # (a re-import wraps it once)
g1_decompress.__wrapped__ = _ORACLE_G1_DECOMPRESS


def register():
    oparams.CURVES.setdefault("bls12_377", BLS12_377)
    omarlin._g1_decompress = g1_decompress
    b2m_testutil.CURVE_ID.setdefault("bls12_377", _lib.CURVE_BLS12_377)
    if "bls12_377" not in opairing._ENGINES:
        opairing._ENGINES["bls12_377"] = Bls377PairingEngine()
    return opairing._ENGINES["bls12_377"]


register()
