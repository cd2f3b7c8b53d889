// ark-serialize G1 points -> affine Montgomery points, host/device shared (the verifier's decode kernel in verify_impl.cuh and
// the SRS loader's in ark_points.cuh run it once per point; tests/ compile it for the host).
//
// ark-serialize 0.3 `CanonicalDeserialize` of a short-Weierstrass affine point in compressed form [U ark-ec
// short_weierstrass_jacobian.rs, ark-serialize SWFlags]: x little-endian in sizeof(Fq) bytes, the two top bits of the last
// byte are flags (bit 7: y is the larger of the two roots, bit 6: the point at infinity; both set is not a flag value).
// y = sqrt(x^3 + b) (fq_sqrt: one exponentiation for BLS12-381 and BN254, Tonelli-Shanks for BLS12-377).  The uncompressed form is x || y with the
// flags in y's last byte; `deserialize_uncompressed` checks x, y < p, and both forms check the curve equation and the
// prime-order subgroup [U].  BN254 G1 has cofactor 1: every curve point passes.  BLS12-381 G1 has a cofactor; its subgroup
// test is the endomorphism one of Scott, "A note on group membership tests for G1, G2 and GT on BLS pairing-friendly curves"
// (2021): with phi(x, y) = (omega x, y), omega a cube root of unity in Fq, P is in G1 iff phi(P) = -u^2 P, u = -0xd201000000010000
// the curve parameter.  That is two multiplications by the 64-bit |u| (126 doublings, 10 additions) instead of r * P
// (255 doublings, ~128 additions); g1_times_r_is_inf keeps the definitional test for the tests.  BLS12-377 G1 uses the same test
// with its own u = 0x8508c00000000001 and omega (u^2 does not depend on the sign of u).  Its b = 1, so x = 0 decompresses to
// (0, +-1), a point of order 3 that the subgroup test rejects.
#pragma once
#include "curve.cuh"
#include "field.cuh"
#include "g2.cuh"

namespace b2m {

// per-point status of the decoders (G2 points use the same codes)
enum : int {
  G1_OK = 0,
  G1_BAD_FLAGS = 1,        // both flag bits set
  G1_X_NOT_CANONICAL = 2,  // x >= p (G2: either component)
  G1_NOT_ON_CURVE = 3,     // compressed: x^3 + b is not a square; uncompressed: y^2 != x^3 + b
  G1_NOT_IN_SUBGROUP = 4,
  G1_Y_NOT_CANONICAL = 5   // uncompressed forms: y >= p (G2: either component)
};

inline const char* point_status_name(int s) {
  switch (s) {
    case G1_OK: return "ok";
    case G1_BAD_FLAGS: return "both flag bits set";
    case G1_X_NOT_CANONICAL: return "x is not below the field modulus";
    case G1_NOT_ON_CURVE: return "not on the curve";
    case G1_NOT_IN_SUBGROUP: return "not in the prime-order subgroup";
    case G1_Y_NOT_CANONICAL: return "y is not below the field modulus";
    default: return "unknown status";
  }
}

template <class Fq>
struct G1Curve;
template <>
struct G1Curve<FqBls> {
  static constexpr uint32_t b = 4;
  static constexpr bool has_cofactor = true;
  using Fr = FrBls;
  static constexpr uint64_t u_abs = 0xd201000000010000ull;
  B2M_HD static FqBls omega() {  // the cube root of unity with phi(g) = -u^2 g for the standard generator g (Montgomery form)
    const uint32_t w[12] = {0x798a64e8u, 0x30f1361bu, 0x7ece5a2au, 0xf3b8ddabu, 0xc61577f7u, 0x16a8ca3au,
                            0x74fd029bu, 0xc26a2ff8u, 0x60701c6eu, 0x3636b766u, 0x241b6160u, 0x051ba4abu};
    FqBls c;
    for (int i = 0; i < 12; i++) c.l[i] = w[i];
    return c;
  }
};
template <>
struct G1Curve<FqBls377> {
  static constexpr uint32_t b = 1;
  static constexpr bool has_cofactor = true;
  using Fr = FrBls377;
  static constexpr uint64_t u_abs = 0x8508c00000000001ull;
  B2M_HD static FqBls377 omega() {  // 2^((q - 1) / 3), the cube root of unity with phi(g) = -u^2 g (Montgomery form)
    const uint32_t w[12] = {0x5a7b8727u, 0x2c766f92u, 0x253d58b5u, 0x03d7f6b0u, 0xec122131u, 0x838ec0deu,
                            0xf658bb10u, 0xbd5eb3e9u, 0x6ed3e52eu, 0x6942bd12u, 0xdd04ed6au, 0x01673786u};
    FqBls377 c;
    for (int i = 0; i < 12; i++) c.l[i] = w[i];
    return c;
  }
};
template <>
struct G1Curve<FqBn> {
  static constexpr uint32_t b = 3;
  static constexpr bool has_cofactor = false;
  using Fr = FrBn;
  static constexpr uint64_t u_abs = 0;
  B2M_HD static FqBn omega() { return FqBn::zero(); }
};

// little-endian bytes -> limbs (no reduction)
template <class Fq>
B2M_HD Fq fq_load(const uint8_t* bytes) {
  Fq x;
  for (int i = 0; i < Fq::N; i++)
    x.l[i] = (uint32_t)bytes[4 * i] | ((uint32_t)bytes[4 * i + 1] << 8) | ((uint32_t)bytes[4 * i + 2] << 16) | ((uint32_t)bytes[4 * i + 3] << 24);
  return x;
}

// canonical limbs < p ?
template <class Fq>
B2M_HD bool fq_below_modulus(const Fq& c) {
  for (int i = Fq::N - 1; i >= 0; i--) {
    const uint32_t m = Fq::Params::mod(i);
    if (c.l[i] != m) return c.l[i] < m;
  }
  return false;
}

// r * P == O: the definitional subgroup test (reference for the tests only)
template <class Fq>
B2M_HD bool g1_times_r_is_inf(const Affine<Fq>& p) {
  uint32_t r[G1Curve<Fq>::Fr::N];
  for (int i = 0; i < G1Curve<Fq>::Fr::N; i++) r[i] = G1Curve<Fq>::Fr::Params::mod(i);
  return scalar_mul<Fq>(p, r, G1Curve<Fq>::Fr::N).is_inf();
}

// P (a finite curve point) in the prime-order subgroup?
template <class Fq>
B2M_HD bool g1_in_subgroup(const Affine<Fq>& p) {
  if (!G1Curve<Fq>::has_cofactor) return true;
  constexpr uint64_t z = G1Curve<Fq>::u_abs;
  const uint32_t zl[2] = {(uint32_t)z, (uint32_t)(z >> 32)};
  const XYZZ<Fq> zp = scalar_mul<Fq>(p, zl, 2);
  XYZZ<Fq> q = zp;  // z * (z * P), double-and-add from the top bit of z
  for (int b = 62; b >= 0; b--) {
    q = q.dbl();
    if ((z >> b) & 1u) q.add(zp);
  }
  if (q.is_inf()) return false;  // u^2 P = O only for points of order dividing u^2, never in G1 \ {O}
  // phi(P) == -q  <=>  omega x * ZZ == X  and  y * ZZZ == -Y
  return (G1Curve<Fq>::omega() * p.x) * q.ZZ == q.X && p.y * q.ZZZ == q.Y.neg();
}

template <class Fq>
B2M_HD int g1_decompress(const uint8_t* bytes, Affine<Fq>* out) {
  constexpr int N = Fq::N;
  Fq x = fq_load<Fq>(bytes);
  const uint32_t flags = x.l[N - 1] >> 30;
  x.l[N - 1] &= 0x3fffffffu;
  *out = Affine<Fq>::inf();
  if (flags == 3u) return G1_BAD_FLAGS;
  if (flags == 1u) return G1_OK;  // infinity
  if (!fq_below_modulus(x)) return G1_X_NOT_CANONICAL;
  const Fq xm = Fq::from_canonical(x);
  const Fq rhs = xm.sqr() * xm + Fq::from_u64(G1Curve<Fq>::b);
  Fq y;
  if (!fq_sqrt(rhs, &y)) return G1_NOT_ON_CURVE;
  const bool larger = y.to_canonical().canonical_gt_half();
  if (larger != (flags == 2u)) y = y.neg();
  const Affine<Fq> p{xm, y};
  if (!g1_in_subgroup(p)) return G1_NOT_IN_SUBGROUP;
  *out = p;
  return G1_OK;
}

// the shared tail of the uncompressed forms: the curve equation and the subgroup; *out = p when both hold
template <class Fq>
B2M_HD int g1_check_store(const Affine<Fq>& p, Affine<Fq>* out) {
  if (p.y.sqr() != p.x.sqr() * p.x + Fq::from_u64(G1Curve<Fq>::b)) return G1_NOT_ON_CURVE;
  if (!g1_in_subgroup(p)) return G1_NOT_IN_SUBGROUP;
  *out = p;
  return G1_OK;
}

// `deserialize_uncompressed` (checked): x || y, flags in y's last byte.  The infinity flag accepts any canonical coordinates,
// as ark-serialize does; the sign bit carries no meaning in this form.
template <class Fq>
B2M_HD int g1_decode_uncompressed(const uint8_t* bytes, Affine<Fq>* out) {
  constexpr int N = Fq::N;
  const Fq x = fq_load<Fq>(bytes);
  Fq y = fq_load<Fq>(bytes + N * 4);
  const uint32_t flags = y.l[N - 1] >> 30;
  y.l[N - 1] &= 0x3fffffffu;
  *out = Affine<Fq>::inf();
  if (flags == 3u) return G1_BAD_FLAGS;
  if (!fq_below_modulus(x)) return G1_X_NOT_CANONICAL;
  if (!fq_below_modulus(y)) return G1_Y_NOT_CANONICAL;
  if (flags & 1u) return G1_OK;  // infinity
  return g1_check_store(Affine<Fq>{Fq::from_canonical(x), Fq::from_canonical(y)}, out);
}

// snarkjs "LEM" form (.ptau files): x || y, each little-endian MONTGOMERY limbs with R = 2^(64 * limbs) -- for these fields
// exactly the device's 32-bit-limb Montgomery form, so no conversion.  No flags: all-zero bytes are the point at infinity
// [U snarkjs].  A limb vector >= p is not a field element (a non-reduced representative) and is rejected.
template <class Fq>
B2M_HD int g1_decode_lem(const uint8_t* bytes, Affine<Fq>* out) {
  constexpr int N = Fq::N;
  const Fq x = fq_load<Fq>(bytes), y = fq_load<Fq>(bytes + N * 4);
  *out = Affine<Fq>::inf();
  if (x.is_zero() && y.is_zero()) return G1_OK;  // infinity ((0, 0) is on none of the curves: b != 0)
  if (!fq_below_modulus(x)) return G1_X_NOT_CANONICAL;
  if (!fq_below_modulus(y)) return G1_Y_NOT_CANONICAL;
  return g1_check_store(Affine<Fq>{x, y}, out);
}

// affine Montgomery -> `serialize` (compressed) bytes: canonical x, bit 7 = y is the larger root, infinity = zero + bit 6
template <class Fq>
B2M_HD void g1_compress(const Affine<Fq>& p, uint8_t* out) {
  constexpr int N = Fq::N;
  Fq x = Fq::zero();
  if (p.is_inf()) {
    x.l[N - 1] = 1u << 30;
  } else {
    x = p.x.to_canonical();
    if (p.y.to_canonical().canonical_gt_half()) x.l[N - 1] |= 1u << 31;
  }
  for (int i = 0; i < N; i++)
    for (int k = 0; k < 4; k++) out[4 * i + k] = (uint8_t)(x.l[i] >> (8 * k));
}

}  // namespace b2m
