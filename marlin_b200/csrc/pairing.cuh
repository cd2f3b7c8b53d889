// Optimal-ate pairing product check, host/device shared: the pairing kernel (pairing_impl.cuh) runs it once per product and
// tests/ compile it for the host.  `PairingEngine::product_of_pairings(pairs).is_one()` [U ark-ec 0.3 bls12 / bn models].
//
// Tower: Fq2 = Fq[u] / (u^2 + beta) (g2.cuh), Fq6 = Fq2[v] / (v^3 - xi), Fq12 = Fq6[w] / (w^2 - v), xi = alpha + u with
// (alpha, beta) = (1, 1) BLS12-381, (9, 1) BN254, (0, 5) BLS12-377 (the PairingParams of pairing_host.hpp).  So w^6 = xi, and an
// Fq12 element is the sum over k = 0..5 of a_k w^k with a_k in Fq2, a_k = c(k % 2).c(k / 2).
//
// G2 points enter as affine twist points over Fq2.  Their line coefficients are computed once per point (g2_lines) in homogeneous
// projective coordinates, three Fq2 values per doubling or addition step, in the form of arkworks' `G2Prepared::ell_coeffs`, and
// evaluated at the affine G1 point without inversions.  M-type twist (BLS12-381, untwisted (x / w^2, y / w^3)): the line,
// times w^3, has terms at 1, w^2 = v and w^3 (mul_by_014).  D-type (BN254, BLS12-377, untwisted (x w^2, y w^3)): terms at 1, w
// and w^3 (mul_by_034).  Vertical lines and Fq2 / Fq4 factors of the lines are dropped: the easy part of the final
// exponentiation maps every element of a proper subfield to 1.
//
// Miller loop: BLS12 over the bits of |x|, conjugated at the end for x < 0 (BLS12-381); BN254 over the NAF of 6u + 2, then
// the lines through pi(Q) and -pi^2(Q).  All pairs of one product share one accumulator.
//
// Final exponentiation: the easy part f^((p^6 - 1)(p^2 + 1)), then a hard part that computes f^(e (p^4 - p^2 + 1) / r):
//   BLS12: (x - 1)^2 (x + p)(x^2 + p^2 - 1) + 3 = 3 (p^4 - p^2 + 1) / r                          e = 3
//   BN254: the chain of Fuentes-Castaneda, Knapp and Rodriguez-Henriquez (arkworks' bn model)   e = 2u (6u^2 + 3u + 1)
// so the pairing computed is the optimal-ate pairing raised to e (r divides neither e): GT values are e-th powers of arkworks'
// (which are not part of the ABI) and "product == 1" is decided exactly.
#pragma once
#include <cstdint>

#include "curve.cuh"
#include "field.cuh"
#include "g1_decode.cuh"
#include "g2.cuh"

// the tower's large operations stay out of line on the device (fully inlined, one pairing is hundreds of thousands of
// instructions and takes minutes to compile)
#ifdef __CUDACC__
#define B2M_PNI __host__ __device__ __noinline__
#else
#define B2M_PNI inline
#endif

namespace b2m {

// Loop constants.  digit(i) of the loop scalar for i below `steps` (the top digit, 1, is implicit in T = Q); `pos` / `neg` are
// the +1 / -1 digits below bit 64.
template <class Fq>
struct AteLoop;
template <>
struct AteLoop<FqBls> {
  static constexpr uint32_t alpha = 1;
  static constexpr int steps = 63;  // |x| = 0xd201000000010000, bit 63 on top
  static constexpr uint64_t pos = 0xd201000000010000ull, neg = 0;
  static constexpr bool x_negative = true, m_twist = true, bn = false;
  static constexpr uint64_t x_abs = 0xd201000000010000ull;
};
template <>
struct AteLoop<FqBls377> {
  static constexpr uint32_t alpha = 0;
  static constexpr int steps = 63;  // x = 0x8508c00000000001
  static constexpr uint64_t pos = 0x8508c00000000001ull, neg = 0;
  static constexpr bool x_negative = false, m_twist = false, bn = false;
  static constexpr uint64_t x_abs = 0x8508c00000000001ull;
};
template <>
struct AteLoop<FqBn> {
  static constexpr uint32_t alpha = 9;
  static constexpr int steps = 65;  // NAF of 6u + 2: 66 digits, the top one at 65, digit 64 is 0
  static constexpr uint64_t pos = 0x2002004200804028ull, neg = 0x82889008420a0480ull;
  static constexpr bool x_negative = false, m_twist = false, bn = true;
  static constexpr uint64_t x_abs = 0x44e992b44a6909f1ull;  // u
};

template <class Fq>
B2M_HD int ate_digit(int i) {
  if (i >= 64) return 0;
  if ((AteLoop<Fq>::pos >> i) & 1u) return 1;
  if ((AteLoop<Fq>::neg >> i) & 1u) return -1;
  return 0;
}

// line steps per G2 point: one doubling per digit, one addition per non-zero digit, BN254's two Frobenius lines
template <class Fq>
__host__ __device__ constexpr int ate_line_count() {
  int n = 0;
  for (int i = AteLoop<Fq>::steps - 1; i >= 0; i--) {
    n++;
    const uint64_t bit = i < 64 ? (1ull << i) : 0;
    if ((AteLoop<Fq>::pos | AteLoop<Fq>::neg) & bit) n++;
  }
  return n + (AteLoop<Fq>::bn ? 2 : 0);
}

// ---- Fq2 helpers ---------------------------------------------------------------------------------------------------------
template <class Fq>
B2M_HD Fq fq_mul_alpha(const Fq& a) {
  constexpr uint32_t al = AteLoop<Fq>::alpha;
  if constexpr (al == 0) return Fq::zero();
  else if constexpr (al == 1) return a;
  else {
    static_assert(al == 9, "alpha");
    return a.dbl().dbl().dbl() + a;
  }
}
// a xi = (a0 + a1 u)(alpha + u) = (alpha a0 - beta a1) + (a0 + alpha a1) u
template <class Fq>
B2M_HD Fq2<Fq> fq2_mul_xi(const Fq2<Fq>& a) {
  return Fq2<Fq>{fq_mul_alpha(a.c0) - Fq2<Fq>::mul_beta(a.c1), a.c0 + fq_mul_alpha(a.c1)};
}
template <class Fq>
B2M_HD Fq2<Fq> fq2_sqr(const Fq2<Fq>& a) {  // (a0 + a1)(a0 - beta a1) - (1 - beta) a0 a1 + 2 a0 a1 u
  const Fq v0 = a.c0 * a.c1;
  return Fq2<Fq>{(a.c0 + a.c1) * (a.c0 - Fq2<Fq>::mul_beta(a.c1)) - v0 + Fq2<Fq>::mul_beta(v0), v0.dbl()};
}
template <class Fq>
B2M_HD Fq2<Fq> fq2_conj(const Fq2<Fq>& a) {
  return Fq2<Fq>{a.c0, a.c1.neg()};
}
template <class Fq>
B2M_HD Fq2<Fq> fq2_scale(const Fq2<Fq>& a, const Fq& k) {
  return Fq2<Fq>{a.c0 * k, a.c1 * k};
}

// ---- Fq6 -------------------------------------------------------------------------------------------------------------------
template <class Fq>
struct Fq6 {
  using F2 = Fq2<Fq>;
  F2 c0, c1, c2;
  B2M_HD static Fq6 zero() { return Fq6{F2::zero(), F2::zero(), F2::zero()}; }
  B2M_HD static Fq6 one() { return Fq6{F2::one(), F2::zero(), F2::zero()}; }
  B2M_HD bool operator==(const Fq6& o) const { return c0 == o.c0 && c1 == o.c1 && c2 == o.c2; }
  B2M_HD friend Fq6 operator+(const Fq6& a, const Fq6& b) { return Fq6{a.c0 + b.c0, a.c1 + b.c1, a.c2 + b.c2}; }
  B2M_HD friend Fq6 operator-(const Fq6& a, const Fq6& b) { return Fq6{a.c0 - b.c0, a.c1 - b.c1, a.c2 - b.c2}; }
  B2M_HD Fq6 neg() const { return Fq6{c0.neg(), c1.neg(), c2.neg()}; }
  B2M_HD Fq6 mul_by_v() const { return Fq6{fq2_mul_xi(c2), c0, c1}; }
};

// Karatsuba
template <class Fq>
B2M_PNI Fq6<Fq> fq6_mul(const Fq6<Fq>& a, const Fq6<Fq>& b) {
  const Fq2<Fq> aa = a.c0 * b.c0, bb = a.c1 * b.c1, cc = a.c2 * b.c2;
  const Fq2<Fq> t1 = fq2_mul_xi((a.c1 + a.c2) * (b.c1 + b.c2) - bb - cc) + aa;
  const Fq2<Fq> t2 = (a.c0 + a.c1) * (b.c0 + b.c1) - aa - bb + fq2_mul_xi(cc);
  const Fq2<Fq> t3 = (a.c0 + a.c2) * (b.c0 + b.c2) - aa + bb - cc;
  return Fq6<Fq>{t1, t2, t3};
}
// Chung-Hasan SQR2
template <class Fq>
B2M_PNI Fq6<Fq> fq6_sqr(const Fq6<Fq>& a) {
  const Fq2<Fq> s0 = fq2_sqr(a.c0), s1 = (a.c0 * a.c1).dbl(), s2 = fq2_sqr(a.c0 - a.c1 + a.c2), s3 = (a.c1 * a.c2).dbl(), s4 = fq2_sqr(a.c2);
  return Fq6<Fq>{s0 + fq2_mul_xi(s3), s1 + fq2_mul_xi(s4), s1 + s2 + s3 - s0 - s4};
}
// a (b0 + b1 v)
template <class Fq>
B2M_PNI Fq6<Fq> fq6_mul_by_01(const Fq6<Fq>& a, const Fq2<Fq>& b0, const Fq2<Fq>& b1) {
  const Fq2<Fq> aa = a.c0 * b0, bb = a.c1 * b1;
  return Fq6<Fq>{fq2_mul_xi(a.c2 * b1) + aa, (b0 + b1) * (a.c0 + a.c1) - aa - bb, a.c2 * b0 + bb};
}
// a b1 v
template <class Fq>
B2M_HD Fq6<Fq> fq6_mul_by_1(const Fq6<Fq>& a, const Fq2<Fq>& b1) {
  return Fq6<Fq>{fq2_mul_xi(a.c2 * b1), a.c0 * b1, a.c1 * b1};
}
template <class Fq>
B2M_HD Fq6<Fq> fq6_scale(const Fq6<Fq>& a, const Fq2<Fq>& k) {
  return Fq6<Fq>{a.c0 * k, a.c1 * k, a.c2 * k};
}
template <class Fq>
B2M_PNI Fq6<Fq> fq6_inverse(const Fq6<Fq>& a) {
  const Fq2<Fq> t0 = fq2_sqr(a.c0) - fq2_mul_xi(a.c1 * a.c2), t1 = fq2_mul_xi(fq2_sqr(a.c2)) - a.c0 * a.c1, t2 = fq2_sqr(a.c1) - a.c0 * a.c2;
  const Fq2<Fq> n = (a.c0 * t0 + fq2_mul_xi(a.c2 * t1 + a.c1 * t2)).inverse();
  return Fq6<Fq>{t0 * n, t1 * n, t2 * n};
}

// ---- Fq12 ------------------------------------------------------------------------------------------------------------------
template <class Fq>
struct Fq12T {
  Fq6<Fq> c0, c1;
  B2M_HD static Fq12T one() { return Fq12T{Fq6<Fq>::one(), Fq6<Fq>::zero()}; }
  B2M_HD bool operator==(const Fq12T& o) const { return c0 == o.c0 && c1 == o.c1; }
  B2M_HD bool is_one() const { return *this == one(); }
  B2M_HD Fq12T conj() const { return Fq12T{c0, c1.neg()}; }  // f^(p^6)
  // a_k, the coefficient of w^k
  B2M_HD Fq2<Fq>& at(int k) {
    Fq6<Fq>& c = k & 1 ? c1 : c0;
    return k < 2 ? c.c0 : k < 4 ? c.c1 : c.c2;
  }
  B2M_HD const Fq2<Fq>& at(int k) const { return const_cast<Fq12T*>(this)->at(k); }
};

template <class Fq>
B2M_PNI Fq12T<Fq> fq12_mul(const Fq12T<Fq>& a, const Fq12T<Fq>& b) {
  const Fq6<Fq> aa = fq6_mul(a.c0, b.c0), bb = fq6_mul(a.c1, b.c1);
  return Fq12T<Fq>{aa + bb.mul_by_v(), fq6_mul(a.c0 + a.c1, b.c0 + b.c1) - aa - bb};
}
// complex squaring: (c0 + c1 w)^2 = (c0 + c1)(c0 + v c1) - (1 + v) c0 c1 + 2 c0 c1 w
template <class Fq>
B2M_PNI Fq12T<Fq> fq12_sqr(const Fq12T<Fq>& a) {
  const Fq6<Fq> ab = fq6_mul(a.c0, a.c1);
  const Fq6<Fq> t = fq6_mul(a.c0 + a.c1, a.c0 + a.c1.mul_by_v()) - ab - ab.mul_by_v();
  return Fq12T<Fq>{t, ab + ab};
}
// f (d0 + d1 v + d4 v w): the M-type line
template <class Fq>
B2M_PNI Fq12T<Fq> fq12_mul_by_014(const Fq12T<Fq>& f, const Fq2<Fq>& d0, const Fq2<Fq>& d1, const Fq2<Fq>& d4) {
  const Fq6<Fq> aa = fq6_mul_by_01(f.c0, d0, d1), bb = fq6_mul_by_1(f.c1, d4);
  const Fq6<Fq> c1 = fq6_mul_by_01(f.c0 + f.c1, d0, d1 + d4) - aa - bb;
  return Fq12T<Fq>{bb.mul_by_v() + aa, c1};
}
// f (d0 + d3 w + d4 v w): the D-type line
template <class Fq>
B2M_PNI Fq12T<Fq> fq12_mul_by_034(const Fq12T<Fq>& f, const Fq2<Fq>& d0, const Fq2<Fq>& d3, const Fq2<Fq>& d4) {
  const Fq6<Fq> aa = fq6_scale(f.c0, d0), bb = fq6_mul_by_01(f.c1, d3, d4);
  const Fq6<Fq> c1 = fq6_mul_by_01(f.c0 + f.c1, d0 + d3, d4) - aa - bb;
  return Fq12T<Fq>{bb.mul_by_v() + aa, c1};
}
// (c0 - c1 w) / (c0^2 - v c1^2): one Fq6, one Fq2 and one Fq inversion
template <class Fq>
B2M_PNI Fq12T<Fq> fq12_inverse(const Fq12T<Fq>& a) {
  const Fq6<Fq> t = fq6_inverse(fq6_sqr(a.c0) - fq6_sqr(a.c1).mul_by_v());
  return Fq12T<Fq>{fq6_mul(a.c0, t), fq6_mul(a.c1, t).neg()};
}
// Granger-Scott squaring, valid in the cyclotomic subgroup (after the easy part): Fq12 as Fq4^3 with Fq4 = Fq2[w^3]
template <class Fq>
B2M_PNI Fq12T<Fq> fq12_cyclotomic_sqr(const Fq12T<Fq>& a) {
  using F2 = Fq2<Fq>;
  F2 z0 = a.c0.c0, z4 = a.c0.c1, z3 = a.c0.c2, z2 = a.c1.c0, z1 = a.c1.c1, z5 = a.c1.c2;
  auto sq4 = [](const F2& x, const F2& y, F2& s0, F2& s1) {  // (x + y w^3)^2 = s0 + s1 w^3
    const F2 t = x * y;
    s0 = (x + y) * (x + fq2_mul_xi(y)) - t - fq2_mul_xi(t);
    s1 = t.dbl();
  };
  F2 t0, t1, t2, t3, t4, t5;
  sq4(z0, z1, t0, t1);
  sq4(z2, z3, t2, t3);
  sq4(z4, z5, t4, t5);
  z0 = (t0 - z0).dbl() + t0;
  z1 = (t1 + z1).dbl() + t1;
  const F2 t = fq2_mul_xi(t5);
  z2 = (t + z2).dbl() + t;
  z3 = (t4 - z3).dbl() + t4;
  z4 = (t2 - z4).dbl() + t2;
  z5 = (t3 + z5).dbl() + t3;
  return Fq12T<Fq>{Fq6<Fq>{z0, z4, z3}, Fq6<Fq>{z2, z1, z5}};
}

// Frobenius coefficients: frob1[k] = xi^(k (p - 1) / 6) (w^k)^p = conj-free factor of w^k, frob2[k] = xi^(k (p^2 - 1) / 6) in Fq.
// Computed once on the host (pairing_consts) and handed to the kernel by value.
template <class Fq>
struct PairingConsts {
  Fq2<Fq> frob1[6];
  Fq frob2[6];
};

// f^p and f^(p^2): a_k -> conj(a_k) frob1[k], a_k -> a_k frob2[k]
template <class Fq>
B2M_PNI Fq12T<Fq> fq12_frobenius1(const Fq12T<Fq>& f, const PairingConsts<Fq>& C) {
  Fq12T<Fq> r;
  for (int k = 0; k < 6; k++) r.at(k) = fq2_conj(f.at(k)) * C.frob1[k];
  return r;
}
template <class Fq>
B2M_PNI Fq12T<Fq> fq12_frobenius2(const Fq12T<Fq>& f, const PairingConsts<Fq>& C) {
  Fq12T<Fq> r;
  for (int k = 0; k < 6; k++) r.at(k) = fq2_scale(f.at(k), C.frob2[k]);
  return r;
}

// f^|x| (|u| for BN254) by cyclotomic square-and-multiply
template <class Fq>
B2M_PNI Fq12T<Fq> fq12_exp_by_x_abs(const Fq12T<Fq>& f) {
  constexpr uint64_t x = AteLoop<Fq>::x_abs;
  int top = 63;
  while (!((x >> top) & 1u)) top--;
  Fq12T<Fq> r = f;
  for (int b = top - 1; b >= 0; b--) {
    r = fq12_cyclotomic_sqr(r);
    if ((x >> b) & 1u) r = fq12_mul(r, f);
  }
  return r;
}
// f^x with the sign of x (BLS12)
template <class Fq>
B2M_HD Fq12T<Fq> fq12_exp_by_x(const Fq12T<Fq>& f) {
  const Fq12T<Fq> r = fq12_exp_by_x_abs(f);
  return AteLoop<Fq>::x_negative ? r.conj() : r;
}

// f^((p^12 - 1) / r * e), e as in the header comment
template <class Fq>
B2M_PNI Fq12T<Fq> final_exponentiation_ate(const Fq12T<Fq>& f, const PairingConsts<Fq>& C) {
  Fq12T<Fq> g = fq12_mul(f.conj(), fq12_inverse(f));  // ^(p^6 - 1)
  g = fq12_mul(fq12_frobenius2(g, C), g);            // ^(p^2 + 1)
  if constexpr (!AteLoop<Fq>::bn) {
    const Fq12T<Fq> t0 = fq12_mul(fq12_exp_by_x(g), g.conj());                                            // g^(x - 1)
    const Fq12T<Fq> t1 = fq12_mul(fq12_exp_by_x(t0), t0.conj());                                          // g^((x - 1)^2)
    const Fq12T<Fq> t2 = fq12_mul(fq12_exp_by_x(t1), fq12_frobenius1(t1, C));                             // t1^(x + p)
    const Fq12T<Fq> t3 = fq12_mul(fq12_mul(fq12_exp_by_x(fq12_exp_by_x(t2)), fq12_frobenius2(t2, C)), t2.conj());  // t2^(x^2 + p^2 - 1)
    return fq12_mul(t3, fq12_mul(fq12_cyclotomic_sqr(g), g));                                            // * g^3
  } else {
    // exponents in the comments, u the BN parameter
    const Fq12T<Fq> a = fq12_exp_by_x_abs(g).conj();        // -u
    const Fq12T<Fq> b = fq12_cyclotomic_sqr(a);              // -2u
    const Fq12T<Fq> d = fq12_mul(fq12_cyclotomic_sqr(b), b);  // -6u
    const Fq12T<Fq> e = fq12_exp_by_x_abs(d).conj();        // 6u^2
    const Fq12T<Fq> h = fq12_exp_by_x_abs(fq12_cyclotomic_sqr(e));  // 12u^3
    const Fq12T<Fq> k = fq12_mul(fq12_mul(h, e), d.conj());  // 12u^3 + 6u^2 + 6u
    const Fq12T<Fq> l = fq12_mul(k, b);                      // 12u^3 + 6u^2 + 4u
    const Fq12T<Fq> n = fq12_mul(fq12_mul(k, e), g);         // 12u^3 + 12u^2 + 6u + 1
    const Fq12T<Fq> r1 = fq12_mul(fq12_mul(fq12_frobenius2(k, C), fq12_frobenius1(l, C)), n);
    const Fq12T<Fq> t = fq12_mul(g.conj(), l);
    return fq12_mul(fq12_frobenius1(fq12_frobenius2(t, C), C), r1);
  }
}

// ---- constants (host) -----------------------------------------------------------------------------------------------------
template <class Fq>
Fq2<Fq> fq2_pow_limbs(const Fq2<Fq>& a, const uint32_t* e, int nlimbs) {
  Fq2<Fq> r = Fq2<Fq>::one();
  for (int i = nlimbs - 1; i >= 0; i--)
    for (int b = 31; b >= 0; b--) {
      r = fq2_sqr(r);
      if ((e[i] >> b) & 1u) r = r * a;
    }
  return r;
}
template <class Fq>
PairingConsts<Fq> pairing_consts() {
  uint32_t e[Fq::N];  // (p - 1) / 6: p = 1 mod 6 for a curve with a sextic twist
  uint64_t rem = 0;
  for (int i = Fq::N - 1; i >= 0; i--) {
    const uint64_t cur = (rem << 32) | (i == 0 ? Fq::Params::mod(0) - 1u : Fq::Params::mod(i));
    e[i] = (uint32_t)(cur / 6);
    rem = cur % 6;
  }
  const Fq2<Fq> xi{Fq::from_u64(AteLoop<Fq>::alpha), Fq::one()};
  const Fq2<Fq> g1 = fq2_pow_limbs(xi, e, Fq::N);                                                    // xi^((p - 1) / 6)
  const Fq g2 = (Fq::from_u64(AteLoop<Fq>::alpha) * Fq::from_u64(AteLoop<Fq>::alpha) + Fq::from_u64(Fq2<Fq>::beta)).pow_limbs(e, Fq::N);  // N(xi)^((p - 1) / 6)
  PairingConsts<Fq> C;
  C.frob1[0] = Fq2<Fq>::one();
  C.frob2[0] = Fq::one();
  for (int k = 1; k < 6; k++) {
    C.frob1[k] = C.frob1[k - 1] * g1;
    C.frob2[k] = C.frob2[k - 1] * g2;
  }
  return C;
}

// ---- prepared G2 -----------------------------------------------------------------------------------------------------------
template <class Fq>
struct G2Line {
  Fq2<Fq> c[3];
};

// The line coefficients of an affine twist point Q (x, y), ate_line_count<Fq>() of them, into `out`.  Q must be finite and on
// the twist; pairs with Q at infinity are left out by the caller.
template <class Fq>
B2M_HD void g2_lines(const Fq2<Fq>& qx, const Fq2<Fq>& qy, const PairingConsts<Fq>& C, G2Line<Fq>* out) {
  using F2 = Fq2<Fq>;
  using L = AteLoop<Fq>;
  F2 X = qx, Y = qy, Z = F2::one();
  const F2 bt = G2Curve<Fq>::b();
  auto half = [](const F2& a) { return F2{fq_halve(a.c0), fq_halve(a.c1)}; };
  int s = 0;
  auto emit = [&](const F2& a, const F2& b, const F2& c) {  // (w^0, v, v w) for M-type, (w^0, w, v w) for D-type
    if (L::m_twist) out[s++] = G2Line<Fq>{{a, b, c}};
    else out[s++] = G2Line<Fq>{{c, b, a}};
  };
  auto dbl = [&]() {
    const F2 a = half(X * Y), b = fq2_sqr(Y), c = fq2_sqr(Z), e = bt * (c.dbl() + c), f = e.dbl() + e, g = half(b + f);
    const F2 h = fq2_sqr(Y + Z) - (b + c), i = e - b, j = fq2_sqr(X), ee = fq2_sqr(e);
    X = a * (b - f);
    Y = fq2_sqr(g) - (ee.dbl() + ee);
    Z = b * h;
    // M: (i, 3j, -h) at (1, v, v w); D: (-h, 3j, i) at (1, w, v w), i.e. emit(i, 3j, -h) in both
    emit(i, j.dbl() + j, h.neg());
  };
  auto add = [&](const F2& x2, const F2& y2) {
    const F2 theta = Y - y2 * Z, lambda = X - x2 * Z, c = fq2_sqr(theta), d = fq2_sqr(lambda), e = lambda * d, f = Z * c, g = X * d;
    const F2 h = e + f - g.dbl();
    X = lambda * h;
    Y = theta * (g - h) - e * Y;
    Z = Z * e;
    // M: (j, -theta, lambda); D: (lambda, -theta, j)
    emit(theta * x2 - lambda * y2, theta.neg(), lambda);
  };
  const F2 nqy = qy.neg();
  for (int i = L::steps - 1; i >= 0; i--) {
    dbl();
    const int d = ate_digit<Fq>(i);
    if (d == 1) add(qx, qy);
    else if (d == -1) add(qx, nqy);
  }
  if constexpr (L::bn) {  // pi(Q) = (conj(x) xi^((p-1)/3), conj(y) xi^((p-1)/2)); -pi^2(Q) = (x xi^((p^2-1)/3), -y xi^((p^2-1)/2))
    add(fq2_conj(qx) * C.frob1[2], fq2_conj(qy) * C.frob1[3]);
    add(fq2_scale(qx, C.frob2[2]), fq2_scale(qy, C.frob2[3]).neg());
  }
}

// ark-serialize uncompressed G2 bytes (x.c0 || x.c1 || y.c0 || y.c1, infinity = bit 6 of the last byte) -> an affine twist point
// or *inf; G1_* status.  Components must be canonical and a finite point must lie on the twist.  No subgroup test: the caller
// decodes untrusted points with b2m_g2_decode_ark, which has one.
template <class Fq>
B2M_HD int g2_affine_uncompressed(const uint8_t* bytes, Fq2<Fq>* x, Fq2<Fq>* y, bool* inf) {
  constexpr int N = Fq::N, NB = Fq::N * 4;
  const Fq x0 = fq_load<Fq>(bytes), x1 = fq_load<Fq>(bytes + NB), y0 = fq_load<Fq>(bytes + 2 * NB);
  Fq y1 = fq_load<Fq>(bytes + 3 * NB);
  const uint32_t flags = y1.l[N - 1] >> 30;
  y1.l[N - 1] &= 0x3fffffffu;
  *inf = true;
  if (flags == 3u) return G1_BAD_FLAGS;
  if (!fq_below_modulus(x0) || !fq_below_modulus(x1)) return G1_X_NOT_CANONICAL;
  if (!fq_below_modulus(y0) || !fq_below_modulus(y1)) return G1_Y_NOT_CANONICAL;
  if (flags & 1u) return G1_OK;
  *x = Fq2<Fq>{Fq::from_canonical(x0), Fq::from_canonical(x1)};
  *y = Fq2<Fq>{Fq::from_canonical(y0), Fq::from_canonical(y1)};
  if (fq2_sqr(*y) != fq2_sqr(*x) * *x + G2Curve<Fq>::b()) return G1_NOT_ON_CURVE;
  *inf = false;
  return G1_OK;
}

// an affine G1 point in Montgomery form ((0, 0) = infinity) with limbs below p and on the curve?
template <class Fq>
B2M_HD bool g1_pairing_input_ok(const Affine<Fq>& p) {
  if (p.is_inf()) return true;
  return fq_below_modulus(p.x) && fq_below_modulus(p.y) && p.y.sqr() == p.x.sqr() * p.x + Fq::from_u64(G1Curve<Fq>::b);
}

// f * line(P) for an affine G1 point P
template <class Fq>
B2M_HD Fq12T<Fq> fq12_mul_line(const Fq12T<Fq>& f, const G2Line<Fq>& l, const Affine<Fq>& p) {
  if constexpr (AteLoop<Fq>::m_twist) return fq12_mul_by_014(f, l.c[0], fq2_scale(l.c[1], p.x), fq2_scale(l.c[2], p.y));
  else return fq12_mul_by_034(f, fq2_scale(l.c[0], p.y), fq2_scale(l.c[1], p.x), l.c[2]);
}

// prod_j f_Q_j(P_j) over n pairs: pair j is the G1 point at(j) with the lines lines(j) (nullptr: Q_j at infinity, the pair is
// skipped; so is P_j at infinity).  at / lines are callables, so the kernel can read pairs straight from global memory.
template <class Fq, class At, class Lines>
B2M_HD Fq12T<Fq> miller_loop_ate(int n, At at, Lines lines) {
  using L = AteLoop<Fq>;
  Fq12T<Fq> f = Fq12T<Fq>::one();
  int s = 0;
  auto step = [&]() {
    for (int j = 0; j < n; j++) {
      const G2Line<Fq>* q = lines(j);
      if (!q) continue;
      const Affine<Fq> p = at(j);
      if (p.is_inf()) continue;
      f = fq12_mul_line(f, q[s], p);
    }
    s++;
  };
  for (int i = L::steps - 1; i >= 0; i--) {
    if (i != L::steps - 1) f = fq12_sqr(f);
    step();
    if (ate_digit<Fq>(i) != 0) step();
  }
  if (L::x_negative) f = f.conj();
  if constexpr (L::bn) {
    step();
    step();
  }
  return f;
}

}  // namespace b2m
