// G2 arithmetic over Fq2, host/device shared: the SRS loader decodes and subgroup-checks G2 points on the GPU (ark_points.cuh),
// the host builds the G2 half of `KZG10::setup` with the same code (g2_host.hpp), and tests/ compile it for the host.
//
// Fq2 = Fq[u] / (u^2 + 1) for both supported curves; E'(Fq2): y^2 = x^3 + b' with b' = 4 (1 + u) (BLS12-381, M-type twist)
// and b' = 3 / (9 + u) (BN254, D-type twist).  The group-law formulas below never need b'.
#pragma once
#include <cstdint>

#include "field.cuh"

namespace b2m {

template <class Fq>
struct Fq2 {
  Fq c0, c1;
  B2M_HD static Fq2 zero() { return Fq2{Fq::zero(), Fq::zero()}; }
  B2M_HD static Fq2 one() { return Fq2{Fq::one(), Fq::zero()}; }
  B2M_HD bool is_zero() const { return c0.is_zero() && c1.is_zero(); }
  B2M_HD bool operator==(const Fq2& o) const { return c0 == o.c0 && c1 == o.c1; }
  B2M_HD bool operator!=(const Fq2& o) const { return !(*this == o); }
  B2M_HD friend Fq2 operator+(const Fq2& a, const Fq2& b) { return Fq2{a.c0 + b.c0, a.c1 + b.c1}; }
  B2M_HD friend Fq2 operator-(const Fq2& a, const Fq2& b) { return Fq2{a.c0 - b.c0, a.c1 - b.c1}; }
  B2M_HD friend Fq2 operator*(const Fq2& a, const Fq2& b) {  // Karatsuba, u^2 = -1
    const Fq v0 = a.c0 * b.c0, v1 = a.c1 * b.c1;
    return Fq2{v0 - v1, (a.c0 + a.c1) * (b.c0 + b.c1) - v0 - v1};
  }
  B2M_HD Fq2 sqr() const { return (*this) * (*this); }
  B2M_HD Fq2 dbl() const { return Fq2{c0.dbl(), c1.dbl()}; }
  B2M_HD Fq2 neg() const { return Fq2{c0.neg(), c1.neg()}; }
  B2M_HD Fq2 inverse() const {  // (c0 - c1 u) / (c0^2 + c1^2)
    const Fq n = (c0.sqr() + c1.sqr()).inverse();
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

// a^((p + 1) / 4), a square root of a when one exists (both base fields are 3 mod 4); true iff it squares back to a
template <class Fq>
B2M_HD bool fq_sqrt(const Fq& a, Fq* out) {
  constexpr int N = Fq::N;
  uint32_t e[N];  // (p + 1) / 4: p = 3 mod 4, so p + 1 carries out of limb 0 only when it is 0xffffffff (never here)
  for (int i = 0; i < N; i++) e[i] = Fq::Params::mod(i);
  e[0] += 1u;
  for (int i = 0; i < N - 1; i++) e[i] = (e[i] >> 2) | (e[i + 1] << 30);
  e[N - 1] >>= 2;
  *out = a.pow_limbs(e, N);
  return out->sqr() == a;
}

// Square root in Fq2 for p = 3 mod 4 by the norm ("complex") method: with n = sqrt(c0^2 + c1^2) in Fq, x = sqrt((c0 +- n) / 2)
// and y = c1 / (2 x) give (x + y u)^2 = c0 + c1 u.  Three Fq exponentiations and one inversion.  False if a is not a square.
template <class Fq>
B2M_HD bool fq2_sqrt(const Fq2<Fq>& a, Fq2<Fq>* out) {
  Fq s;
  if (a.c1.is_zero()) {
    if (fq_sqrt(a.c0, &s)) {
      *out = Fq2<Fq>{s, Fq::zero()};
      return true;
    }
    if (fq_sqrt(a.c0.neg(), &s)) {  // (s u)^2 = -s^2
      *out = Fq2<Fq>{Fq::zero(), s};
      return true;
    }
    return false;
  }
  Fq n;
  if (!fq_sqrt(a.c0.sqr() + a.c1.sqr(), &n)) return false;
  Fq x;
  if (!fq_sqrt(fq_halve(a.c0 + n), &x) && !fq_sqrt(fq_halve(a.c0 - n), &x)) return false;
  *out = Fq2<Fq>{x, a.c1 * x.dbl().inverse_fast()};
  return out->sqr() == a;
}

}  // namespace b2m
