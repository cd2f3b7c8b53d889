// Host build of the .ptau point decoders of g1_decode.cuh / g2_decode.cuh (snarkjs LEM form), the bodies of the LEM decode
// kernels, over a tiny C ABI for tests/test_ptau_host.py.  curve: 0 = BLS12-381, 1 = BN254.
#include "../../marlin_b200/csrc/g2_decode.cuh"
using namespace b2m;

template <class Fq>
static void g1_lem(const uint8_t* bytes, int n, uint32_t* out, int* status) {
  for (int i = 0; i < n; i++) {
    Affine<Fq> p;
    status[i] = g1_decode_lem<Fq>(bytes + (size_t)i * 2 * Fq::N * 4, &p);
    memcpy(out + (size_t)i * 2 * Fq::N, &p, sizeof(p));
  }
}
extern "C" void g1_decode_lem_host(int curve, const uint8_t* bytes, int n, uint32_t* out, int* status) {
  if (curve == 0) g1_lem<FqBls>(bytes, n, out, status);
  else g1_lem<FqBn>(bytes, n, out, status);
}

template <class Fq>
static void g2_lem(const uint8_t* bytes, int n, uint8_t* out, int* status) {
  for (int i = 0; i < n; i++) status[i] = g2_decode_lem<Fq>(bytes + (size_t)i * 4 * Fq::N * 4, out + (size_t)i * 4 * Fq::N * 4);
}
extern "C" void g2_decode_lem_host(int curve, const uint8_t* bytes, int n, uint8_t* out, int* status) {
  if (curve == 0) g2_lem<FqBls>(bytes, n, out, status);
  else g2_lem<FqBn>(bytes, n, out, status);
}
