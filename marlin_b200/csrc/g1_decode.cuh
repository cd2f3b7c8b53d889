// Compressed G1 points of a proof -> affine Montgomery points, host/device shared (the verifier's decode kernel in
// verify_impl.cuh runs it once per point; tests/ compile it for the host).
//
// ark-serialize 0.3 `CanonicalDeserialize` of a short-Weierstrass affine point in compressed form [U ark-ec
// short_weierstrass_jacobian.rs, ark-serialize SWFlags]: x little-endian in sizeof(Fq) bytes, the two top bits of the last
// byte are flags (bit 7: y is the larger of the two roots, bit 6: the point at infinity; both set is not a flag value).
// y = (x^3 + b)^((p + 1) / 4) (both base fields are 3 mod 4), checked by squaring.  ark-serialize 0.3 `deserialize` also
// checks the prime-order subgroup [U]; BLS12-381 G1 has a cofactor, so a point of that curve must satisfy r * P = O
// (BN254 G1 has cofactor 1: every curve point passes).
#pragma once
#include "curve.cuh"
#include "field.cuh"

namespace b2m {

enum : int {
  G1_OK = 0,
  G1_BAD_FLAGS = 1,     // both flag bits set
  G1_X_NOT_CANONICAL = 2,  // x >= p
  G1_NOT_ON_CURVE = 3,  // x^3 + b is not a square
  G1_NOT_IN_SUBGROUP = 4
};

template <class Fq>
struct G1Curve;
template <>
struct G1Curve<FqBls> {
  static constexpr uint32_t b = 4;
  static constexpr bool has_cofactor = true;
  using Fr = FrBls;
};
template <>
struct G1Curve<FqBn> {
  static constexpr uint32_t b = 3;
  static constexpr bool has_cofactor = false;
  using Fr = FrBn;
};

template <class Fq>
B2M_HD int g1_decompress(const uint8_t* bytes, Affine<Fq>* out) {
  constexpr int N = Fq::N;
  Fq x;
  for (int i = 0; i < N; i++)
    x.l[i] = (uint32_t)bytes[4 * i] | ((uint32_t)bytes[4 * i + 1] << 8) | ((uint32_t)bytes[4 * i + 2] << 16) | ((uint32_t)bytes[4 * i + 3] << 24);
  const uint32_t flags = x.l[N - 1] >> 30;
  x.l[N - 1] &= 0x3fffffffu;
  *out = Affine<Fq>::inf();
  if (flags == 3u) return G1_BAD_FLAGS;
  if (flags == 1u) return G1_OK;  // infinity
  for (int i = N - 1; i >= 0; i--) {  // x < p
    const uint32_t m = Fq::Params::mod(i);
    if (x.l[i] != m) {
      if (x.l[i] > m) return G1_X_NOT_CANONICAL;
      break;
    }
    if (i == 0) return G1_X_NOT_CANONICAL;
  }
  const Fq xm = Fq::from_canonical(x);
  const Fq rhs = xm.sqr() * xm + Fq::from_u64(G1Curve<Fq>::b);
  uint32_t e[N];  // (p + 1) / 4: p = 3 mod 4, so p + 1 carries out of limb 0 only when it is 0xffffffff (never here)
  for (int i = 0; i < N; i++) e[i] = Fq::Params::mod(i);
  e[0] += 1u;
  for (int i = 0; i < N - 1; i++) e[i] = (e[i] >> 2) | (e[i + 1] << 30);
  e[N - 1] >>= 2;
  Fq y = rhs.pow_limbs(e, N);
  if (y.sqr() != rhs) return G1_NOT_ON_CURVE;
  const bool larger = y.to_canonical().canonical_gt_half();
  if (larger != (flags == 2u)) y = y.neg();
  const Affine<Fq> p{xm, y};
  if (G1Curve<Fq>::has_cofactor) {
    uint32_t r[G1Curve<Fq>::Fr::N];
    for (int i = 0; i < G1Curve<Fq>::Fr::N; i++) r[i] = G1Curve<Fq>::Fr::Params::mod(i);
    if (!scalar_mul<Fq>(p, r, G1Curve<Fq>::Fr::N).is_inf()) return G1_NOT_IN_SUBGROUP;
  }
  *out = p;
  return G1_OK;
}

}  // namespace b2m
