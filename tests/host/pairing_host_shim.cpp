// Host build of the optimal-ate pairing (pairing.cuh) next to the reduced Tate pairing of pairing_host.hpp, over a tiny C ABI
// for tests/test_pairing_host.py.  curve: 0 BLS12-381, 1 BN254, 2 BLS12-377 (the C ABI's ids).  G1 points cross the ABI as
// canonical little-endian 32-bit limbs x || y ((0, 0) = infinity), G2 points as ark-serialize uncompressed bytes.
#include <vector>

#include "../../marlin_b200/csrc/pairing.cuh"
#include "../../marlin_b200/csrc/pairing_host.hpp"
using namespace b2m;

template <class Fq>
static Fq load(const uint32_t* a) {
  Fq x;
  memcpy(x.l, a, sizeof(x.l));
  return Fq::from_canonical(x);
}
template <class Fq>
static Affine<Fq> load_g1(const uint32_t* pp) {
  bool inf = true;
  for (int k = 0; k < 2 * Fq::N; k++) inf = inf && pp[k] == 0;
  return inf ? Affine<Fq>::inf() : Affine<Fq>{load<Fq>(pp), load<Fq>(pp + Fq::N)};
}

// mode 0: *ok = optimal-ate product == 1; mode 1: also out = the product's GT value as 12 canonical Fq coefficients of
// 1, w, ..., w^11 (the basis of pairing_host.hpp's single extension, u = w^6 - alpha); mode 2: *ok = Tate product == 1.
// -1 for a G2 input that is malformed or off the twist, -2 for a G1 input off the curve.
template <class Fq>
static int run(int mode, int n, const uint32_t* pts, const uint8_t* g2, int* ok, uint32_t* out) {
  const PairingConsts<Fq> C = pairing_consts<Fq>();
  constexpr int NL = ate_line_count<Fq>();
  std::vector<G2Line<Fq>> lines((size_t)n * NL);
  std::vector<char> g2inf(n);
  std::vector<Affine<Fq>> p(n);
  for (int i = 0; i < n; i++) {
    Fq2<Fq> x, y;
    bool inf;
    if (g2_affine_uncompressed<Fq>(g2 + (size_t)i * 4 * Fq::N * 4, &x, &y, &inf) != G1_OK) return -1;
    g2inf[i] = inf;
    if (!inf) g2_lines<Fq>(x, y, C, lines.data() + (size_t)i * NL);
    p[i] = load_g1<Fq>(pts + (size_t)i * 2 * Fq::N);
    if (!g1_pairing_input_ok(p[i])) return -2;
  }
  if (mode == 2) {
    std::vector<G2Prepared<Fq>> q(n);
    std::vector<std::pair<Affine<Fq>, const G2Prepared<Fq>*>> pairs;
    for (int i = 0; i < n; i++) {
      if (g2inf[i]) continue;
      if (!g2_prepare<Fq>(g2 + (size_t)i * 4 * Fq::N * 4, &q[i])) return -1;
      pairs.push_back({p[i], &q[i]});
    }
    *ok = pairing_product_is_one(pairs) ? 1 : 0;
    return 0;
  }
  const Fq12T<Fq> f = miller_loop_ate<Fq>(
      n, [&](int j) { return p[j]; }, [&](int j) { return g2inf[j] ? nullptr : lines.data() + (size_t)j * NL; });
  const Fq12T<Fq> e = final_exponentiation_ate(f, C);
  *ok = e.is_one() ? 1 : 0;
  if (mode == 1) {
    Fq c[12];
    for (auto& x : c) x = Fq::zero();
    const Fq alpha = Fq::from_u64(AteLoop<Fq>::alpha);
    for (int k = 0; k < 6; k++) {  // a_k w^k = (x + y u) w^k = (x - alpha y) w^k + y w^(k + 6)
      c[k] = e.at(k).c0 - alpha * e.at(k).c1;
      c[k + 6] = e.at(k).c1;
    }
    for (int k = 0; k < 12; k++) {
      const Fq v = c[k].to_canonical();
      memcpy(out + k * Fq::N, v.l, sizeof(v.l));
    }
  }
  return 0;
}

extern "C" int pairing_product(int curve, int mode, int n, const uint32_t* pts, const uint8_t* g2, int* ok, uint32_t* out) {
  switch (curve) {
    case 0: return run<FqBls>(mode, n, pts, g2, ok, out);
    case 1: return run<FqBn>(mode, n, pts, g2, ok, out);
    default: return run<FqBls377>(mode, n, pts, g2, ok, out);
  }
}

extern "C" int ate_lines_per_point(int curve) {
  return curve == 0 ? ate_line_count<FqBls>() : curve == 1 ? ate_line_count<FqBn>() : ate_line_count<FqBls377>();
}
