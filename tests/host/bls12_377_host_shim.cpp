// Host build of the BLS12-377 instantiation of the device arithmetic -- Fr / Fq (field.cuh), Tonelli-Shanks and the beta = 5
// Fq2 (g2.cuh), G1 / G2 decoding and the endomorphism subgroup test (g1_decode.cuh, g2_decode.cuh) and the host pairing
// (pairing_host.hpp) -- over a tiny C ABI for tests/test_bls12_377_host.py.  All field elements cross the ABI as canonical
// little-endian 32-bit limbs.
#include "../../marlin_b200/csrc/g2_decode.cuh"
#include "../../marlin_b200/csrc/pairing_host.hpp"
using namespace b2m;
using Fr = FrBls377;
using Fq = FqBls377;

template <class F>
static F load(const uint32_t* a) {
  F x;
  memcpy(x.l, a, sizeof(x.l));
  return F::from_canonical(x);
}
template <class F>
static void store(const F& x, uint32_t* r) {
  const F c = x.to_canonical();
  memcpy(r, c.l, sizeof(c.l));
}

// which: 0 a * b, 1 a + b, 2 a - b, 3 Fermat inverse, 4 binary-Euclid inverse, 5 sqrt (returns 1 iff a is a square)
template <class F>
static int op(int which, const uint32_t* a, const uint32_t* b, uint32_t* r) {
  const F x = load<F>(a), y = load<F>(b);
  F z = F::zero();
  int ok = 1;
  switch (which) {
    case 0: z = x * y; break;
    case 1: z = x + y; break;
    case 2: z = x - y; break;
    case 3: z = x.inverse(); break;
    case 4: z = x.inverse_fast(); break;
    case 5:
      if constexpr (F::N == 12) ok = fq_sqrt(x, &z);
      break;
  }
  store(z, r);
  return ok;
}
extern "C" int field_op(int field, int which, const uint32_t* a, const uint32_t* b, uint32_t* r) {
  return field == 0 ? op<Fr>(which, a, b, r) : op<Fq>(which, a, b, r);
}

// Fq2 (c0 || c1): which 0 a * b, 1 a^-1, 2 sqrt (returns 1 iff a is a square)
extern "C" int fq2_op(int which, const uint32_t* a, const uint32_t* b, uint32_t* r) {
  const Fq2<Fq> x{load<Fq>(a), load<Fq>(a + Fq::N)}, y{load<Fq>(b), load<Fq>(b + Fq::N)};
  Fq2<Fq> z = Fq2<Fq>::zero();
  int ok = 1;
  switch (which) {
    case 0: z = x * y; break;
    case 1: z = x.inverse(); break;
    case 2: ok = fq2_sqrt(x, &z); break;
  }
  store(z.c0, r);
  store(z.c1, r + Fq::N);
  return ok;
}

// n G1 points in either ark-serialize form -> canonical affine x || y limbs (infinity: 0, 0) and a G1_* status each
extern "C" void g1_decode_host(const uint8_t* bytes, int n, int compressed, uint32_t* out, int* status) {
  const size_t pb = (compressed ? 1 : 2) * Fq::N * 4;
  for (int i = 0; i < n; i++) {
    Affine<Fq> p;
    status[i] = compressed ? g1_decompress<Fq>(bytes + i * pb, &p) : g1_decode_uncompressed<Fq>(bytes + i * pb, &p);
    if (p.is_inf()) p = Affine<Fq>{Fq::zero(), Fq::zero()};
    else p = Affine<Fq>{p.x.to_canonical(), p.y.to_canonical()};
    memcpy(out + (size_t)i * 2 * Fq::N, &p, sizeof(p));
  }
}

// canonical affine points assumed on the curve: out[2i] = endomorphism test, out[2i + 1] = (r * P == O)
extern "C" void g1_subgroup_host(const uint32_t* pts, int n, int* out) {
  for (int i = 0; i < n; i++) {
    const Affine<Fq> p{load<Fq>(pts + (size_t)i * 2 * Fq::N), load<Fq>(pts + (size_t)i * 2 * Fq::N + Fq::N)};
    out[2 * i] = g1_in_subgroup(p);
    out[2 * i + 1] = g1_times_r_is_inf(p);
  }
}

// n G2 points in either form -> uncompressed canonical bytes and a status each
extern "C" void g2_decode_host(const uint8_t* bytes, int n, int compressed, uint8_t* out, int* status) {
  const size_t pb = (compressed ? 2 : 4) * Fq::N * 4;
  for (int i = 0; i < n; i++) status[i] = g2_decode<Fq>(bytes + i * pb, compressed != 0, out + (size_t)i * 4 * Fq::N * 4);
}

// the reduced pairing of canonical G1 points with uncompressed G2 points: mode 0: *ok = (product == 1); mode 1: out = the
// value of the first pair, 12 canonical Fq coefficients of the basis 1, w, ..., w^11.  -1 for a G2 input off the twist.
extern "C" int pairing_host(int mode, int n, const uint32_t* pts, const uint8_t* g2, int* ok, uint32_t* out) {
  std::vector<G2Prepared<Fq>> q(n);
  std::vector<std::pair<Affine<Fq>, const G2Prepared<Fq>*>> pairs;
  for (int i = 0; i < n; i++) {
    if (!g2_prepare<Fq>(g2 + (size_t)i * 4 * Fq::N * 4, &q[i])) return -1;
    const uint32_t* pp = pts + (size_t)i * 2 * Fq::N;
    bool inf = true;
    for (int k = 0; k < 2 * Fq::N; k++) inf = inf && pp[k] == 0;
    pairs.push_back({inf ? Affine<Fq>::inf() : Affine<Fq>{load<Fq>(pp), load<Fq>(pp + Fq::N)}, &q[i]});
  }
  if (mode == 0) {
    *ok = pairing_product_is_one(pairs) ? 1 : 0;
  } else {
    const Fq12<Fq> v = final_exponentiation(miller_loop(pairs));
    for (int k = 0; k < 12; k++) store(v.c[k], out + k * Fq::N);
  }
  return 0;
}
