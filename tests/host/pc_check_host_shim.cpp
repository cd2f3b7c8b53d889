// Host build of the Level-1 check's bookkeeping (marlin_b200/csrc/pc_check.hpp) over a tiny C ABI for tests/test_pc_check_host.py.
#include "../../marlin_b200/csrc/pc_check.hpp"
using namespace b2m;

// a: b2m_pc_check_combinations's 19 array arguments after n_sets, in order.  Set s of n: its pc_set_error (into err, return -2),
// else pc_set_equations with the set's points at base0 (-1 malformed).  On success out receives per point: n_plain, n_bounded,
// the plain terms (base, 8 u32 Montgomery limbs of c), the bounded terms (bound index, base, c), z (8 u32) and w; returns the
// number of u32 words written.
template <class Fr>
static long terms(int pc, size_t n, const void* const* a, size_t s, const uint64_t* bounds, size_t n_bounds, uint32_t base0, uint32_t* out,
                  char* err, size_t err_cap) {
  const PcSets S{n, (const size_t*)a[0], (const uint8_t*)a[1], (const int64_t*)a[2], (const int*)a[3], (const uint8_t*)a[4],
                 (const size_t*)a[5], (const size_t*)a[6], (const int64_t*)a[7], (const uint64_t*)a[8], (const size_t*)a[9],
                 (const uint64_t*)a[10], (const uint8_t*)a[11], (const int*)a[12], (const uint8_t*)a[13], (const size_t*)a[14],
                 (const size_t*)a[15], (const size_t*)a[16], (const uint8_t*)a[17], (const uint64_t*)a[18]};
  const std::vector<uint64_t> b(bounds, bounds + n_bounds);
  const std::string e = pc_set_error<Fr>(S, s, b);
  if (!e.empty()) {
    snprintf(err, err_cap, "%s", e.c_str());
    return -2;
  }
  VerifyEq<Fr> E;
  if (!pc_set_equations<Fr>(pc, S, s, b, base0, E)) return -1;
  long o = 0;
  auto put = [&](const Fr& x) {
    for (int i = 0; i < Fr::N; i++) out[o++] = x.l[i];
  };
  for (const auto& pe : E.pt) {
    out[o++] = (uint32_t)pe.plain.size();
    out[o++] = (uint32_t)pe.bounded.size();
    for (const auto& t : pe.plain) {
      out[o++] = t.base;
      put(t.c);
    }
    for (const auto& t : pe.bounded) {
      out[o++] = (uint32_t)t.first;
      out[o++] = t.second.base;
      put(t.second.c);
    }
    put(pe.z);
    out[o++] = pe.w;
  }
  return o;
}

extern "C" long pc_terms_host(int curve, int pc, size_t n, const void* const* arrays, size_t s, const uint64_t* bounds, size_t n_bounds,
                              uint32_t base0, uint32_t* out, char* err, size_t err_cap) {
  if (curve == B2M_CURVE_BLS12_381) return terms<FrBls>(pc, n, arrays, s, bounds, n_bounds, base0, out, err, err_cap);
  return terms<FrBn>(pc, n, arrays, s, bounds, n_bounds, base0, out, err, err_cap);
}

// Set s's point slots, as pointers relative to the arrays: kind (0 commitment, 1 shifted, 2 w) and index in that array
extern "C" size_t pc_points_host(int pc, size_t n, const void* const* a, size_t s, size_t fq_bytes, uint32_t* kind, uint64_t* index) {
  PcSets S{};
  S.n = n;
  S.comm_off = (const size_t*)a[0];
  S.comms = (const uint8_t*)a[1];
  S.comm_bounds = (const int64_t*)a[2];
  S.has_shifted = (const int*)a[3];
  S.shifted = (const uint8_t*)a[4];
  S.point_off = (const size_t*)a[9];
  S.w = (const uint8_t*)a[11];
  const std::vector<const uint8_t*> p = pc_set_points(pc, S, s, fq_bytes);
  const uint8_t* base[3] = {S.comms, S.shifted, S.w};
  for (size_t i = 0; i < p.size(); i++) {  // the three arrays are separate allocations: a slot lies in exactly one of them
    kind[i] = p[i] >= S.w && p[i] < S.w + fq_bytes * S.point_off[n] ? 2 : (p[i] >= S.shifted && p[i] < S.shifted + fq_bytes * S.comm_off[n] ? 1 : 0);
    index[i] = (p[i] - base[kind[i]]) / fq_bytes;
  }
  return p.size();
}
