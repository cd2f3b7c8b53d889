// Host build of the verifier's shared code -- the compressed-G1 decoder (marlin_b200/csrc/g1_decode.cuh, the body of the
// decode kernel) and the pairing product check (pairing_host.hpp) -- over a tiny C ABI for tests/test_verify_host.py.
#include "../../marlin_b200/csrc/g1_decode.cuh"
#include "../../marlin_b200/csrc/pairing_host.hpp"
using namespace b2m;

template <class Fq>
static void decode(const uint8_t* bytes, int n, uint32_t* out, int* status) {
  for (int i = 0; i < n; i++) {
    Affine<Fq> p;
    status[i] = g1_decompress<Fq>(bytes + (size_t)i * Fq::N * 4, &p);
    memcpy(out + (size_t)i * 2 * Fq::N, &p, sizeof(p));
  }
}
extern "C" void g1_decode_host(int curve, const uint8_t* bytes, int n, uint32_t* out, int* status) {
  if (curve == 0) decode<FqBls>(bytes, n, out, status);
  else decode<FqBn>(bytes, n, out, status);
}

// pts: n affine G1 points (Montgomery limbs, (0,0) = infinity); g2: n uncompressed G2 points.  mode 0: *ok = (product == 1);
// mode 1: out = the reduced pairing value of the first pair (12 Fq coefficients, Montgomery).  Returns -1 for a bad G2 input.
template <class Fq>
static int pairing(int mode, int n, const uint32_t* pts, const uint8_t* g2, int* ok, uint32_t* out) {
  std::vector<G2Prepared<Fq>> q(n);
  std::vector<std::pair<Affine<Fq>, const G2Prepared<Fq>*>> pairs;
  for (int i = 0; i < n; i++) {
    if (!g2_prepare<Fq>(g2 + (size_t)i * 4 * Fq::N * 4, &q[i])) return -1;
    Affine<Fq> p;
    memcpy(&p, pts + (size_t)i * 2 * Fq::N, sizeof(p));
    pairs.push_back({p, &q[i]});
  }
  if (mode == 0) {
    *ok = pairing_product_is_one(pairs) ? 1 : 0;
  } else {
    const Fq12<Fq> v = final_exponentiation(miller_loop(pairs));
    memcpy(out, v.c, sizeof(v.c));
  }
  return 0;
}
extern "C" int pairing_host(int curve, int mode, int n, const uint32_t* pts, const uint8_t* g2, int* ok, uint32_t* out) {
  return curve == 0 ? pairing<FqBls>(mode, n, pts, g2, ok, out) : pairing<FqBn>(mode, n, pts, g2, ok, out);
}
