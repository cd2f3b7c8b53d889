// Host-side pairing product check for the batched verifier (verify_impl.cuh): `Π e(P_i, Q_i) == 1`, the final step of
// `KZG10::check` / `batch_check` behind `PC::check_combinations` [reference src/lib.rs:413; U ark-poly-commit kzg10].
// A randomised batch folds every proof into 2 (MarlinKZG10) or 2 + #bounds (SonicKZG10) pairs, so the count per batch is
// constant; like g2_host.hpp this is a handful of operations per call on the CPU with the device's limb code (field.cuh
// compiled for the host), not a fallback for per-proof work.
//
// Only "product == 1" is ever asked, so any non-degenerate bilinear pairing serves.  This is the reduced Tate pairing
// over the single extension
//     Fq12 = Fq[w] / (w^12 - 2 alpha w^6 + alpha^2 + beta)     (w^6 = xi = alpha + u, u^2 = -beta)
// with (alpha, beta) = (1, 1) (BLS12-381), (9, 1) (BN254) or (0, 5) (BLS12-377).  G2 points (on the twist over Fq2) are mapped
// into E(Fq12) by the untwisting isomorphism: M-type (BLS12-381, y^2 = x^3 + b xi): (x, y) -> (x / w^2, y / w^3); D-type
// (BN254, BLS12-377, y^2 = x^3 + b / xi): (x, y) -> (x w^2, y w^3).  The Miller loop runs over the bits of r with lines through multiples of the G1 argument
// (slopes in Fq, vertical lines dropped: they die in the final exponentiation), all pairs sharing one accumulator;
// the final exponentiation is (p^6 - 1)(p^2 + 1) through the Frobenius map, then the hard part (p^4 - p^2 + 1) / r by
// square-and-multiply.
#pragma once
#include <cstdint>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

#include "curve.cuh"
#include "field.cuh"

namespace b2m {

template <class Fq>
struct PairingParams;
template <>
struct PairingParams<FqBls> {
  using Fr = FrBls;
  static constexpr uint64_t alpha = 1, beta = 1, b = 4;
  static constexpr bool m_twist = true;
  // (p^4 - p^2 + 1) / r
  static const char* hard_exp() {
    return "f686b3d807d01c0bd38c3195c899ed3cde88eeb996ca394506632528d6a9a2f230063cf081517f68f7764c28b6f8ae5a72bce8d63cb9f827eca0ba621315b2076995003fc"
           "77a17988f8761bdc51dc2378b9039096d1b767f17fcbde783765915c97f36c6f18212ed0b283ed237db421d160aeb6a1e79983774940996754c8c71a2629b0dea236905ce"
           "937335d5b68fa9912aae208ccf1e516c3f438e3ba79";
  }
};
template <>
struct PairingParams<FqBn> {
  using Fr = FrBn;
  static constexpr uint64_t alpha = 9, beta = 1, b = 3;
  static constexpr bool m_twist = false;
  static const char* hard_exp() {
    return "1baaa710b0759ad331ec15183177faf6c0eb522d5b122784e529a5861876f6b3b1b1355d189227d79581e16f3fd90c66b887d56d5095f23aaa441e3954bcf8adcc7b44c"
           "87cdbacff1154e7e1da014fd5abf5cc4f49c36d4e81bb482ccdf42b1";
  }
};
template <>
struct PairingParams<FqBls377> {
  using Fr = FrBls377;
  static constexpr uint64_t alpha = 0, beta = 5, b = 1;
  static constexpr bool m_twist = false;
  static const char* hard_exp() {
    return "6d616e43720774d7d810d5cbdf0576728e56efc3bf3b4074a5448da5cfbef98d9c2cce3b25c548afd84225b34ccc65eca9c9678a845497a9781d8129911a8d889"
           "828282015fcd1c3fa1470f8b2d1eefd89535f9b5aaae0551dffcf72fb0bd948d5f4548283abcaf63f0a34fcb827dc8f4db069bf65f4f6974b4ff0fa27719b834b"
           "6904468768c0eaeea22e68002e16ba88600000000000000000000001";
  }
};

// little-endian 32-bit limbs of a big-endian hex string
inline std::vector<uint32_t> hex_limbs(const char* hex) {
  const size_t len = strlen(hex);
  std::vector<uint32_t> out((len + 7) / 8, 0u);
  for (size_t i = 0; i < len; i++) {
    const char ch = hex[len - 1 - i];
    const uint32_t v = ch >= 'a' ? ch - 'a' + 10 : ch - '0';
    out[i / 8] |= v << (4 * (i % 8));
  }
  return out;
}

// canonical little-endian limbs < p ?
template <class F>
B2M_HD bool canonical_lt_modulus(const F& c) {
  for (int i = F::N - 1; i >= 0; i--) {
    const uint32_t m = F::Params::mod(i);
    if (c.l[i] != m) return c.l[i] < m;
  }
  return false;
}

template <class Fq>
struct Fq12 {
  Fq c[12];
  static Fq12 zero() {
    Fq12 r;
    for (auto& x : r.c) x = Fq::zero();
    return r;
  }
  static Fq12 one() {
    Fq12 r = zero();
    r.c[0] = Fq::one();
    return r;
  }
  static Fq12 from_fq2(const Fq& a, const Fq& b) {  // a + b u, u = w^6 - alpha
    Fq12 r = zero();
    r.c[0] = a - Fq::from_u64(PairingParams<Fq>::alpha) * b;
    r.c[6] = b;
    return r;
  }
  bool operator==(const Fq12& o) const {
    for (int i = 0; i < 12; i++)
      if (c[i] != o.c[i]) return false;
    return true;
  }
  friend Fq12 operator+(const Fq12& a, const Fq12& b) {
    Fq12 r;
    for (int i = 0; i < 12; i++) r.c[i] = a.c[i] + b.c[i];
    return r;
  }
  friend Fq12 operator-(const Fq12& a, const Fq12& b) {
    Fq12 r;
    for (int i = 0; i < 12; i++) r.c[i] = a.c[i] - b.c[i];
    return r;
  }
  Fq12 scale(const Fq& k) const {
    Fq12 r;
    for (int i = 0; i < 12; i++) r.c[i] = c[i] * k;
    return r;
  }
  // schoolbook product, zero coefficients skipped (the Miller loop's lines have five), reduced with w^12 = c6 w^6 - c0
  // (c6 = 2 alpha, c0 = alpha^2 + beta)
  friend Fq12 operator*(const Fq12& a, const Fq12& b) {
    Fq t[23];
    for (auto& x : t) x = Fq::zero();
    int nzb[12], nb = 0;
    for (int j = 0; j < 12; j++)
      if (!b.c[j].is_zero()) nzb[nb++] = j;
    for (int i = 0; i < 12; i++) {
      if (a.c[i].is_zero()) continue;
      for (int k = 0; k < nb; k++) t[i + nzb[k]] = t[i + nzb[k]] + a.c[i] * b.c[nzb[k]];
    }
    const Fq c6 = Fq::from_u64(2 * PairingParams<Fq>::alpha), c0 = Fq::from_u64(PairingParams<Fq>::alpha * PairingParams<Fq>::alpha + PairingParams<Fq>::beta);
    for (int k = 22; k >= 12; k--) {
      if (t[k].is_zero()) continue;
      t[k - 6] = t[k - 6] + c6 * t[k];
      t[k - 12] = t[k - 12] - c0 * t[k];
    }
    Fq12 r;
    for (int i = 0; i < 12; i++) r.c[i] = t[i];
    return r;
  }
  Fq12 pow(const uint32_t* e, size_t nlimbs) const {
    Fq12 r = one();
    bool started = false;
    for (size_t i = nlimbs; i-- > 0;)
      for (int bit = 31; bit >= 0; bit--) {
        if (started) r = r * r;
        if ((e[i] >> bit) & 1u) {
          r = started ? r * (*this) : *this;
          started = true;
        }
      }
    return r;
  }
};

// Constants of one curve's Fq12, built once: the untwisting factors and the Frobenius images (w^p)^i of the basis.
template <class Fq>
struct PairingTables {
  Fq12<Fq> fx, fy;       // multiply untwisted x / y coordinates by these
  Fq12<Fq> frob[12];     // frob[i] = (w^i)^p
  std::vector<uint32_t> hard;
  static const PairingTables& get() {
    static const PairingTables t;
    return t;
  }
  PairingTables() {
    using E = Fq12<Fq>;
    E w = E::zero();
    w.c[1] = Fq::one();
    E w2 = w * w, w3 = w2 * w;
    if (PairingParams<Fq>::m_twist) {  // w^-1 = (c6 w^5 - w^11) / c0
      const Fq c0 = Fq::from_u64(PairingParams<Fq>::alpha * PairingParams<Fq>::alpha + PairingParams<Fq>::beta);
      E wi = E::zero();
      wi.c[5] = Fq::from_u64(2 * PairingParams<Fq>::alpha);
      wi.c[11] = Fq::one().neg();
      wi = wi.scale(c0.inverse());
      fx = wi * wi;
      fy = fx * wi;
    } else {
      fx = w2;
      fy = w3;
    }
    uint32_t pl[Fq::N];
    for (int i = 0; i < Fq::N; i++) pl[i] = Fq::Params::mod(i);
    const E wp = w.pow(pl, Fq::N);
    frob[0] = E::one();
    for (int i = 1; i < 12; i++) frob[i] = frob[i - 1] * wp;
    hard = hex_limbs(PairingParams<Fq>::hard_exp());
  }
};

template <class Fq>
Fq12<Fq> fq12_frobenius(const Fq12<Fq>& f, int times) {
  const PairingTables<Fq>& T = PairingTables<Fq>::get();
  Fq12<Fq> cur = f;
  for (int k = 0; k < times; k++) {
    Fq12<Fq> r = Fq12<Fq>::zero();
    for (int i = 0; i < 12; i++)
      if (!cur.c[i].is_zero()) r = r + T.frob[i].scale(cur.c[i]);
    cur = r;
  }
  return cur;
}

// f^-1 = (prod_{i=1..11} f^(p^i)) / N(f), the norm N(f) = prod_{i=0..11} f^(p^i) lying in Fq
template <class Fq>
Fq12<Fq> fq12_inverse(const Fq12<Fq>& f) {
  Fq12<Fq> conj = Fq12<Fq>::one(), fi = f;
  for (int i = 1; i < 12; i++) {
    fi = fq12_frobenius(fi, 1);
    conj = conj * fi;
  }
  const Fq n = (conj * f).c[0];
  return conj.scale(n.inverse());
}

// f^((p^12 - 1) / r)
template <class Fq>
Fq12<Fq> final_exponentiation(const Fq12<Fq>& f) {
  Fq12<Fq> u = fq12_frobenius(f, 6) * fq12_inverse(f);  // ^(p^6 - 1)
  u = fq12_frobenius(u, 2) * u;                          // ^(p^2 + 1)
  const std::vector<uint32_t>& h = PairingTables<Fq>::get().hard;
  return u.pow(h.data(), h.size());
}

// A G2 point carried in E(Fq12) coordinates (the image of the untwisting map).
template <class Fq>
struct G2Prepared {
  Fq12<Fq> x, y;
};

// ark-serialize `serialize_uncompressed` bytes of a G2 affine point (x.c0 || x.c1 || y.c0 || y.c1, canonical little-endian,
// infinity flag = bit 6 of the last byte) -> E(Fq12).  False for a coordinate >= p, the point at infinity or a point off
// the twist (checked as y^2 = x^3 + b after untwisting, which is the same equation).
template <class Fq>
bool g2_prepare(const uint8_t* bytes, G2Prepared<Fq>* out) {
  const size_t nb = Fq::N * 4;
  Fq parts[4];
  for (int k = 0; k < 4; k++) {
    Fq c;
    memcpy(c.l, bytes + k * nb, nb);
    if (k == 3) {
      if ((c.l[Fq::N - 1] >> 30) & 1u) return false;
      c.l[Fq::N - 1] &= 0x7fffffffu;  // (bit 7 carries no meaning in the uncompressed form)
    }
    if (!canonical_lt_modulus(c)) return false;
    parts[k] = Fq::from_canonical(c);
  }
  const PairingTables<Fq>& T = PairingTables<Fq>::get();
  out->x = Fq12<Fq>::from_fq2(parts[0], parts[1]) * T.fx;
  out->y = Fq12<Fq>::from_fq2(parts[2], parts[3]) * T.fy;
  Fq12<Fq> rhs = out->x * out->x * out->x;
  rhs.c[0] = rhs.c[0] + Fq::from_u64(PairingParams<Fq>::b);
  return out->y * out->y == rhs;
}

// prod_i f_{r, P_i}(Q_i): one shared accumulator, one squaring per bit of r.  P_i must have order r (or be infinity,
// which contributes 1).
template <class Fq>
Fq12<Fq> miller_loop(const std::vector<std::pair<Affine<Fq>, const G2Prepared<Fq>*>>& pairs) {
  using Fr = typename PairingParams<Fq>::Fr;
  using E = Fq12<Fq>;
  struct St {
    Fq xp, yp, tx, ty;
    const G2Prepared<Fq>* q;
  };
  std::vector<St> st;
  for (const auto& pq : pairs)
    if (!pq.first.is_inf()) st.push_back(St{pq.first.x, pq.first.y, pq.first.x, pq.first.y, pq.second});
  E f = E::one();
  if (st.empty()) return f;
  int top = Fr::N * 32 - 1;
  while (!((Fr::Params::mod(top / 32) >> (top % 32)) & 1u)) top--;
  auto line = [](const St& s, const Fq& lam) {  // (yq - ty) - lam (xq - tx)
    E l = s.q->y - s.q->x.scale(lam);
    l.c[0] = l.c[0] + lam * s.tx - s.ty;
    return l;
  };
  for (int bit = top - 1; bit >= 0; bit--) {
    f = f * f;
    for (St& s : st) {
      const Fq xx = s.tx.sqr();
      const Fq lam = (xx.dbl() + xx) * s.ty.dbl().inverse_fast();
      f = f * line(s, lam);
      const Fq nx = lam.sqr() - s.tx.dbl();
      s.ty = lam * (s.tx - nx) - s.ty;
      s.tx = nx;
    }
    if ((Fr::Params::mod(bit / 32) >> (bit % 32)) & 1u) {
      for (St& s : st) {
        if (s.tx == s.xp) continue;  // T = -P on the last bit: vertical line, T + P = infinity
        const Fq lam = (s.ty - s.yp) * (s.tx - s.xp).inverse_fast();
        f = f * line(s, lam);
        const Fq nx = lam.sqr() - s.tx - s.xp;
        s.ty = lam * (s.tx - nx) - s.ty;
        s.tx = nx;
      }
    }
  }
  return f;
}

template <class Fq>
bool pairing_product_is_one(const std::vector<std::pair<Affine<Fq>, const G2Prepared<Fq>*>>& pairs) {
  return final_exponentiation(miller_loop(pairs)) == Fq12<Fq>::one();
}

}  // namespace b2m
