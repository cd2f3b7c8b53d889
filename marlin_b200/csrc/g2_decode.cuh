// ark-serialize G2 points -> checked uncompressed canonical bytes, host/device shared (the SRS loader's decode kernel in
// ark_points.cuh runs it once per point; tests/ compile it for the host).
//
// Encoding [U ark-serialize / ark-ff 0.3 QuadExtField]: an Fq2 element is c0 || c1, each canonical little-endian in
// sizeof(Fq) bytes.  Compressed: x, with the SWFlags bits in the top of c1's last byte (bit 7: y is the larger root, bit 6:
// infinity).  "Larger" is QuadExtField's ordering: c1 is compared first, then c0.  Uncompressed: x || y with the flags in the
// top of y.c1's last byte -- exactly what g2_write_uncompressed (g2_host.hpp) writes, and the form pairing_host.hpp and
// b2m_vk_create take.  Both forms check every component < p, the twist equation and the subgroup; G2 has a cofactor on both
// curves, so the subgroup test is r * Q = O.  Status codes are g1_decode.cuh's.
#pragma once
#include "g1_decode.cuh"
#include "g2.cuh"

namespace b2m {

// y > -y in QuadExtField's ordering (canonical components)
template <class Fq>
B2M_HD bool fq2_canonical_gt_neg(const Fq& c0, const Fq& c1) {
  return c1.is_zero() ? c0.canonical_gt_half() : c1.canonical_gt_half();
}

template <class Fq>
B2M_HD bool g2_in_subgroup(const Fq2<Fq>& x, const Fq2<Fq>& y) {
  using Fr = typename G1Curve<Fq>::Fr;
  uint32_t r[Fr::N];
  for (int i = 0; i < Fr::N; i++) r[i] = Fr::Params::mod(i);
  return G2Jac<Fq>::mul_affine(x, y, r, Fr::N).is_inf();
}

template <class Fq>
B2M_HD void g2_store_uncompressed(const Fq2<Fq>& x, const Fq2<Fq>& y, bool inf, uint8_t* out) {
  constexpr int N = Fq::N;
  Fq parts[4] = {x.c0, x.c1, y.c0, y.c1};
  for (int k = 0; k < 4; k++) {
    Fq c = inf ? Fq::zero() : parts[k].to_canonical();
    if (inf && k == 3) c.l[N - 1] = 1u << 30;
    for (int i = 0; i < N; i++)
      for (int j = 0; j < 4; j++) out[(k * N + i) * 4 + j] = (uint8_t)(c.l[i] >> (8 * j));
  }
}

// one point in either form -> 4 * sizeof(Fq) uncompressed canonical bytes (infinity: zero coordinates + bit 6); G1_* status
template <class Fq>
B2M_HD int g2_decode(const uint8_t* bytes, bool compressed, uint8_t* out) {
  constexpr int N = Fq::N, NB = Fq::N * 4;
  const Fq x0 = fq_load<Fq>(bytes);
  Fq x1 = fq_load<Fq>(bytes + NB), y0, y1;
  Fq& last = compressed ? x1 : y1;
  if (!compressed) {
    y0 = fq_load<Fq>(bytes + 2 * NB);
    y1 = fq_load<Fq>(bytes + 3 * NB);
  }
  const uint32_t flags = last.l[N - 1] >> 30;
  last.l[N - 1] &= 0x3fffffffu;
  const Fq2<Fq> zero = Fq2<Fq>::zero();
  g2_store_uncompressed<Fq>(zero, zero, true, out);
  if (flags == 3u) return G1_BAD_FLAGS;
  if (!fq_below_modulus(x0) || !fq_below_modulus(x1)) return G1_X_NOT_CANONICAL;
  if (!compressed && (!fq_below_modulus(y0) || !fq_below_modulus(y1))) return G1_Y_NOT_CANONICAL;
  if (flags & 1u) return G1_OK;  // infinity
  const Fq2<Fq> x{Fq::from_canonical(x0), Fq::from_canonical(x1)};
  const Fq2<Fq> rhs = x.sqr() * x + G2Curve<Fq>::b();
  Fq2<Fq> y;
  if (compressed) {
    if (!fq2_sqrt(rhs, &y)) return G1_NOT_ON_CURVE;
    if (fq2_canonical_gt_neg(y.c0.to_canonical(), y.c1.to_canonical()) != (flags == 2u)) y = y.neg();
  } else {
    y = Fq2<Fq>{Fq::from_canonical(y0), Fq::from_canonical(y1)};
    if (y.sqr() != rhs) return G1_NOT_ON_CURVE;
  }
  if (!g2_in_subgroup(x, y)) return G1_NOT_IN_SUBGROUP;
  g2_store_uncompressed<Fq>(x, y, false, out);
  return G1_OK;
}

// snarkjs "LEM" form: x.c0 || x.c1 || y.c0 || y.c1, each little-endian Montgomery limbs (g1_decode_lem); all-zero bytes are
// infinity.  -> uncompressed canonical bytes as g2_decode writes them
template <class Fq>
B2M_HD int g2_decode_lem(const uint8_t* bytes, uint8_t* out) {
  constexpr int NB = Fq::N * 4;
  const Fq x0 = fq_load<Fq>(bytes), x1 = fq_load<Fq>(bytes + NB), y0 = fq_load<Fq>(bytes + 2 * NB), y1 = fq_load<Fq>(bytes + 3 * NB);
  const Fq2<Fq> zero = Fq2<Fq>::zero();
  g2_store_uncompressed<Fq>(zero, zero, true, out);
  if (x0.is_zero() && x1.is_zero() && y0.is_zero() && y1.is_zero()) return G1_OK;  // infinity
  if (!fq_below_modulus(x0) || !fq_below_modulus(x1)) return G1_X_NOT_CANONICAL;
  if (!fq_below_modulus(y0) || !fq_below_modulus(y1)) return G1_Y_NOT_CANONICAL;
  const Fq2<Fq> x{x0, x1}, y{y0, y1};
  if (y.sqr() != x.sqr() * x + G2Curve<Fq>::b()) return G1_NOT_ON_CURVE;
  if (!g2_in_subgroup(x, y)) return G1_NOT_IN_SUBGROUP;
  g2_store_uncompressed<Fq>(x, y, false, out);
  return G1_OK;
}

// uncompressed canonical bytes (as g2_decode writes them) -> compressed bytes; no field multiplication needed
template <class Fq>
B2M_HD void g2_compress(const uint8_t* in, uint8_t* out) {
  constexpr int N = Fq::N, NB = Fq::N * 4;
  Fq x0 = fq_load<Fq>(in), x1 = fq_load<Fq>(in + NB), y0 = fq_load<Fq>(in + 2 * NB), y1 = fq_load<Fq>(in + 3 * NB);
  const bool inf = (y1.l[N - 1] >> 30) & 1u;
  y1.l[N - 1] &= 0x3fffffffu;
  if (inf) {
    x0 = Fq::zero();
    x1 = Fq::zero();
    x1.l[N - 1] = 1u << 30;
  } else if (fq2_canonical_gt_neg(y0, y1)) {
    x1.l[N - 1] |= 1u << 31;
  }
  for (int i = 0; i < N; i++)
    for (int j = 0; j < 4; j++) {
      out[i * 4 + j] = (uint8_t)(x0.l[i] >> (8 * j));
      out[NB + i * 4 + j] = (uint8_t)(x1.l[i] >> (8 * j));
    }
}

}  // namespace b2m
