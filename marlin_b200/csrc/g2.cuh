// G2 arithmetic over Fq2, host/device shared: the SRS loader decodes and subgroup-checks G2 points on the GPU (ark_points.cuh),
// the host builds the G2 half of `KZG10::setup` with the same code (g2_host.hpp), and tests/ compile it for the host.
//
// Fq2 = Fq[u] / (u^2 + beta): beta = 1 for BLS12-381 and BN254, 5 for BLS12-377.  E'(Fq2): y^2 = x^3 + b' with
// b' = 4 (1 + u) (BLS12-381, M-type twist), b' = 3 / (9 + u) (BN254, D-type twist) and b' = 1 / u (BLS12-377, D-type twist).
// The group-law formulas below never need b'.
#pragma once
#include <cstdint>

#include "field.cuh"

namespace b2m {

// beta of Fq2 = Fq[u] / (u^2 + beta)
template <class Fq>
struct Fq2Beta {
  static constexpr uint32_t value = 1;
};
template <>
struct Fq2Beta<FqBls377> {
  static constexpr uint32_t value = 5;
};

template <class Fq>
struct Fq2 {
  static constexpr uint32_t beta = Fq2Beta<Fq>::value;
  static_assert(beta == 1 || beta == 5, "Fq2: u^2 = -1 or -5");
  Fq c0, c1;
  B2M_HD static Fq mul_beta(const Fq& a) {
    if constexpr (beta == 1) return a;
    else return a.dbl().dbl() + a;
  }
  B2M_HD static Fq2 zero() { return Fq2{Fq::zero(), Fq::zero()}; }
  B2M_HD static Fq2 one() { return Fq2{Fq::one(), Fq::zero()}; }
  B2M_HD bool is_zero() const { return c0.is_zero() && c1.is_zero(); }
  B2M_HD bool operator==(const Fq2& o) const { return c0 == o.c0 && c1 == o.c1; }
  B2M_HD bool operator!=(const Fq2& o) const { return !(*this == o); }
  B2M_HD friend Fq2 operator+(const Fq2& a, const Fq2& b) { return Fq2{a.c0 + b.c0, a.c1 + b.c1}; }
  B2M_HD friend Fq2 operator-(const Fq2& a, const Fq2& b) { return Fq2{a.c0 - b.c0, a.c1 - b.c1}; }
  B2M_HD friend Fq2 operator*(const Fq2& a, const Fq2& b) {  // Karatsuba, u^2 = -beta
    const Fq v0 = a.c0 * b.c0, v1 = a.c1 * b.c1;
    return Fq2{v0 - mul_beta(v1), (a.c0 + a.c1) * (b.c0 + b.c1) - v0 - v1};
  }
  B2M_HD Fq2 sqr() const { return (*this) * (*this); }
  B2M_HD Fq2 dbl() const { return Fq2{c0.dbl(), c1.dbl()}; }
  B2M_HD Fq2 neg() const { return Fq2{c0.neg(), c1.neg()}; }
  B2M_HD Fq2 inverse() const {  // (c0 - c1 u) / (c0^2 + beta c1^2)
    const Fq n = (c0.sqr() + mul_beta(c1.sqr())).inverse();
    return Fq2{c0 * n, (c1 * n).neg()};
  }
};

template <class Fq>
struct G2Jac {  // Jacobian: (X / Z^2, Y / Z^3); infinity: Z = 0
  Fq2<Fq> X, Y, Z;
  B2M_HD static G2Jac inf() { return G2Jac{Fq2<Fq>::one(), Fq2<Fq>::one(), Fq2<Fq>::zero()}; }
  B2M_HD bool is_inf() const { return Z.is_zero(); }
  B2M_HD G2Jac dbl() const {  // dbl-2009-l (a = 0)
    if (is_inf()) return *this;
    const Fq2<Fq> A = X.sqr(), B = Y.sqr(), C = B.sqr();
    const Fq2<Fq> D = ((X + B).sqr() - A - C).dbl();
    const Fq2<Fq> E = A.dbl() + A, F = E.sqr();
    G2Jac r;
    r.X = F - D.dbl();
    r.Y = E * (D - r.X) - C.dbl().dbl().dbl();
    r.Z = (Y * Z).dbl();
    return r;
  }
  B2M_HD G2Jac add(const G2Jac& o) const {  // add-2007-bl
    if (is_inf()) return o;
    if (o.is_inf()) return *this;
    const Fq2<Fq> Z1Z1 = Z.sqr(), Z2Z2 = o.Z.sqr();
    const Fq2<Fq> U1 = X * Z2Z2, U2 = o.X * Z1Z1;
    const Fq2<Fq> S1 = Y * o.Z * Z2Z2, S2 = o.Y * Z * Z1Z1;
    if (U1 == U2) return S1 == S2 ? dbl() : inf();
    const Fq2<Fq> H = U2 - U1, I = H.dbl().sqr(), J = H * I, rr = (S2 - S1).dbl(), V = U1 * I;
    G2Jac r;
    r.X = rr.sqr() - J - V.dbl();
    r.Y = rr * (V - r.X) - (S1 * J).dbl();
    r.Z = ((Z + o.Z).sqr() - Z1Z1 - Z2Z2) * H;
    return r;
  }
  // canonical little-endian scalar of nlimbs 32-bit limbs
  B2M_HD G2Jac mul(const uint32_t* k, int nlimbs) const {
    G2Jac acc = inf();
    for (int i = nlimbs - 1; i >= 0; i--)
      for (int b = 31; b >= 0; b--) {
        acc = acc.dbl();
        if ((k[i] >> b) & 1u) acc = acc.add(*this);
      }
    return acc;
  }
  // this + (x2, y2) for a finite affine point (madd-2007-bl): fewer live temporaries than add(), which keeps the GPU's
  // subgroup check of a G2 point in registers
  B2M_HD G2Jac add_affine(const Fq2<Fq>& x2, const Fq2<Fq>& y2) const {
    if (is_inf()) return G2Jac{x2, y2, Fq2<Fq>::one()};
    const Fq2<Fq> Z1Z1 = Z.sqr();
    const Fq2<Fq> H = x2 * Z1Z1 - X, rr = (y2 * Z * Z1Z1 - Y).dbl();
    if (H.is_zero()) return rr.is_zero() ? dbl() : inf();
    const Fq2<Fq> HH = H.sqr(), I = HH.dbl().dbl(), J = H * I, V = X * I;
    G2Jac r;
    r.X = rr.sqr() - J - V.dbl();
    r.Y = rr * (V - r.X) - (Y * J).dbl();
    r.Z = (Z + H).sqr() - Z1Z1 - HH;
    return r;
  }
  // k * (x, y) for a finite affine point, double-and-add from the top set bit
  B2M_HD static G2Jac mul_affine(const Fq2<Fq>& x, const Fq2<Fq>& y, const uint32_t* k, int nlimbs) {
    G2Jac acc = inf();
    bool started = false;
    for (int i = nlimbs - 1; i >= 0; i--)
      for (int b = 31; b >= 0; b--) {
        if (started) acc = acc.dbl();
        if ((k[i] >> b) & 1u) {
          acc = acc.add_affine(x, y);
          started = true;
        }
      }
    return acc;
  }
  B2M_HD void to_affine(Fq2<Fq>* x, Fq2<Fq>* y) const {  // (finite points only)
    const Fq2<Fq> zi = Z.inverse(), zi2 = zi.sqr();
    *x = X * zi2;
    *y = Y * zi2 * zi;
  }
};

// b' of the twist, Montgomery form
template <class Fq>
struct G2Curve;
template <>
struct G2Curve<FqBls> {
  B2M_HD static Fq2<FqBls> b() {  // 4 + 4u
    const uint32_t four[12] = {0x000cfff3u, 0xaa270000u, 0xfc34000au, 0x53cc0032u, 0x6b0a807fu, 0x478fe97au,
                               0xe6ba24d7u, 0xb1d37ebeu, 0xbf78ab2fu, 0x8ec9733bu, 0x3d83de7eu, 0x09d64551u};
    FqBls c;
    for (int i = 0; i < 12; i++) c.l[i] = four[i];
    return Fq2<FqBls>{c, c};
  }
};
template <>
struct G2Curve<FqBn> {
  B2M_HD static Fq2<FqBn> b() {  // 3 / (9 + u) = (27 - 3u) / 82
    const uint32_t c0[8] = {0x77b802a8u, 0x3bf938e3u, 0x3633535du, 0x020b1b27u, 0x49755260u, 0x26b7edf0u, 0x4384a86du, 0x2514c632u};
    const uint32_t c1[8] = {0xd1dcff67u, 0x38e7ecccu, 0x93ce0d3eu, 0x65f0b37du, 0x22ac00aau, 0xd749d0ddu, 0x4a688d4du, 0x0141b9ceu};
    Fq2<FqBn> r;
    for (int i = 0; i < 8; i++) {
      r.c0.l[i] = c0[i];
      r.c1.l[i] = c1[i];
    }
    return r;
  }
};
template <>
struct G2Curve<FqBls377> {
  B2M_HD static Fq2<FqBls377> b() {  // 1 / u = -u / 5
    const uint32_t c1[12] = {0x66666685u, 0x80722666u, 0x899999a9u, 0x8df55926u, 0xd64f34cfu, 0x7fe4561au,
                             0xb6e4f01bu, 0xb95da6d8u, 0xfc142743u, 0x4b747cccu, 0x70f49f43u, 0x0039c3fau};
    Fq2<FqBls377> r{FqBls377::zero(), FqBls377::zero()};
    for (int i = 0; i < 12; i++) r.c1.l[i] = c1[i];
    return r;
  }
};

// a / 2 (the Montgomery form halves like the value: p is odd and below 2^(32N - 1), so a + p never carries out)
template <class Fq>
B2M_HD Fq fq_halve(const Fq& a) {
  Fq t = a;
  if (t.l[0] & 1u) {
    t.l[0] = add_cc(t.l[0], Fq::Params::mod(0));
    for (int i = 1; i < Fq::N - 1; i++) t.l[i] = addc_cc(t.l[i], Fq::Params::mod(i));
    t.l[Fq::N - 1] = addc(t.l[Fq::N - 1], Fq::Params::mod(Fq::N - 1));
  }
  for (int i = 0; i < Fq::N - 1; i++) t.l[i] = (t.l[i] >> 1) | (t.l[i + 1] << 31);
  t.l[Fq::N - 1] >>= 1;
  return t;
}

// A square root of a when one exists; true iff a is a square.  p = 3 mod 4 (TWO_ADICITY 1: BLS12-381, BN254): a^((p + 1) / 4),
// checked by squaring.  Otherwise (BLS12-377: p - 1 = 2^46 t) Tonelli-Shanks with the 2^s-th root of unity g^t of the field's
// non-residue generator g: x = a^((t + 1) / 2), b = a^t; while b != 1, find the least k with b^(2^k) = 1 (k = m means a is not
// a square), then x *= c^(2^(m - k - 1)), c = that squared, b *= c, m = k.  One exponentiation plus at most s (s + 1) / 2 squarings.
template <class Fq>
B2M_HD bool fq_sqrt(const Fq& a, Fq* out) {
  constexpr int N = Fq::N;
  if constexpr (Fq::Params::TWO_ADICITY == 1) {
    uint32_t e[N];  // (p + 1) / 4: p = 3 mod 4, so p + 1 carries out of limb 0 only when it is 0xffffffff (never here)
    for (int i = 0; i < N; i++) e[i] = Fq::Params::mod(i);
    e[0] += 1u;
    for (int i = 0; i < N - 1; i++) e[i] = (e[i] >> 2) | (e[i + 1] << 30);
    e[N - 1] >>= 2;
    *out = a.pow_limbs(e, N);
    return out->sqr() == a;
  } else {
    if (a.is_zero()) {
      *out = a;
      return true;
    }
    uint32_t e[N];
    for (int i = 0; i < N; i++) e[i] = Fq::Params::odd_half(i);
    const Fq w = a.pow_limbs(e, N);  // a^((t - 1) / 2)
    Fq x = a * w, b = x * w, c;
    for (int i = 0; i < N; i++) c.l[i] = Fq::Params::root(i);
    const Fq one = Fq::one();
    int m = Fq::Params::TWO_ADICITY;
    while (b != one) {
      int k = 0;
      for (Fq b2 = b; b2 != one; b2 = b2.sqr())
        if (++k == m) return false;
      for (int j = 0; j < m - k - 1; j++) c = c.sqr();
      x = x * c;
      c = c.sqr();
      b = b * c;
      m = k;
    }
    *out = x;
    return true;
  }
}

// a / beta (beta = 1: a itself)
template <class Fq>
B2M_HD Fq fq2_div_beta(const Fq& a) {
  if constexpr (Fq2<Fq>::beta == 1) return a;
  else return a * Fq::from_u64(Fq2<Fq>::beta).inverse();
}

// Square root in Fq2 by the norm ("complex") method: with n = sqrt(c0^2 + beta c1^2) in Fq, x = sqrt((c0 +- n) / 2) and
// y = c1 / (2 x) give (x + y u)^2 = x^2 - beta y^2 + 2 x y u = c0 + c1 u.  Three Fq square roots and one inversion.  False if
// a is not a square.
template <class Fq>
B2M_HD bool fq2_sqrt(const Fq2<Fq>& a, Fq2<Fq>* out) {
  Fq s;
  if (a.c1.is_zero()) {
    if (fq_sqrt(a.c0, &s)) {
      *out = Fq2<Fq>{s, Fq::zero()};
      return true;
    }
    if (fq_sqrt(fq2_div_beta<Fq>(a.c0.neg()), &s)) {  // (s u)^2 = -beta s^2
      *out = Fq2<Fq>{Fq::zero(), s};
      return true;
    }
    return false;
  }
  Fq n;
  if (!fq_sqrt(a.c0.sqr() + Fq2<Fq>::mul_beta(a.c1.sqr()), &n)) return false;
  Fq x;
  if (!fq_sqrt(fq_halve(a.c0 + n), &x) && !fq_sqrt(fq_halve(a.c0 - n), &x)) return false;
  *out = Fq2<Fq>{x, a.c1 * x.dbl().inverse_fast()};
  return out->sqr() == a;
}

}  // namespace b2m
