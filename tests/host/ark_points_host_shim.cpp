// Host build of the SRS loader's shared point code -- g1_decode.cuh (both G1 forms, the endomorphism subgroup test, G1
// compression) and g2_decode.cuh (both G2 forms, G2 compression) -- over a tiny C ABI for tests/test_ark_srs_host.py.
#include "../../marlin_b200/csrc/g2_decode.cuh"
using namespace b2m;

template <class Fq>
static void g1_decode(const uint8_t* bytes, int n, int compressed, uint32_t* out, int* status) {
  const size_t pb = (compressed ? 1 : 2) * Fq::N * 4;
  for (int i = 0; i < n; i++) {
    Affine<Fq> p;
    status[i] = compressed ? g1_decompress<Fq>(bytes + i * pb, &p) : g1_decode_uncompressed<Fq>(bytes + i * pb, &p);
    memcpy(out + (size_t)i * 2 * Fq::N, &p, sizeof(p));
  }
}
extern "C" void g1_decode_ark_host(int curve, const uint8_t* bytes, int n, int compressed, uint32_t* out, int* status) {
  if (curve == 0) g1_decode<FqBls>(bytes, n, compressed, out, status);
  else g1_decode<FqBn>(bytes, n, compressed, out, status);
}

// pts: n affine Montgomery points assumed on the curve.  out[2i] = endomorphism test, out[2i + 1] = (r * P == O)
template <class Fq>
static void subgroup(const uint32_t* pts, int n, int* out) {
  for (int i = 0; i < n; i++) {
    Affine<Fq> p;
    memcpy(&p, pts + (size_t)i * 2 * Fq::N, sizeof(p));
    out[2 * i] = p.is_inf() || g1_in_subgroup(p);
    out[2 * i + 1] = g1_times_r_is_inf(p);
  }
}
extern "C" void g1_subgroup_host(int curve, const uint32_t* pts, int n, int* out) {
  if (curve == 0) subgroup<FqBls>(pts, n, out);
  else subgroup<FqBn>(pts, n, out);
}

template <class Fq>
static void g1_comp(const uint32_t* pts, int n, uint8_t* out) {
  for (int i = 0; i < n; i++) {
    Affine<Fq> p;
    memcpy(&p, pts + (size_t)i * 2 * Fq::N, sizeof(p));
    g1_compress<Fq>(p, out + (size_t)i * Fq::N * 4);
  }
}
extern "C" void g1_compress_host(int curve, const uint32_t* pts, int n, uint8_t* out) {
  if (curve == 0) g1_comp<FqBls>(pts, n, out);
  else g1_comp<FqBn>(pts, n, out);
}

template <class Fq>
static void g2_dec(const uint8_t* bytes, int n, int compressed, uint8_t* out, int* status) {
  const size_t pb = (compressed ? 2 : 4) * Fq::N * 4;
  for (int i = 0; i < n; i++) status[i] = g2_decode<Fq>(bytes + i * pb, compressed != 0, out + (size_t)i * 4 * Fq::N * 4);
}
extern "C" void g2_decode_ark_host(int curve, const uint8_t* bytes, int n, int compressed, uint8_t* out, int* status) {
  if (curve == 0) g2_dec<FqBls>(bytes, n, compressed, out, status);
  else g2_dec<FqBn>(bytes, n, compressed, out, status);
}

extern "C" void g2_compress_host(int curve, const uint8_t* in, int n, uint8_t* out) {
  for (int i = 0; i < n; i++) {
    if (curve == 0) g2_compress<FqBls>(in + (size_t)i * 4 * FqBls::N * 4, out + (size_t)i * 2 * FqBls::N * 4);
    else g2_compress<FqBn>(in + (size_t)i * 4 * FqBn::N * 4, out + (size_t)i * 2 * FqBn::N * 4);
  }
}
