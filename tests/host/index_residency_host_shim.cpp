// Host build of marlin_b200/csrc/msm_layout.hpp's residency rule and its device- and host-resident byte models, for
// tests/test_index_residency_host.py.
#include "../../marlin_b200/csrc/msm_layout.hpp"

using namespace b2m;

static MsmKeyShape shape_of(size_t n_g, int fr_bits, size_t fq_bytes, int levels) {
  MsmKeyShape k;
  k.n_g = n_g;
  k.n_extra = 3;
  k.fr_bits = fr_bits;
  k.fq_bytes = fq_bytes;
  k.affine_levels = levels;
  return k;
}

extern "C" {
// out = {c, W, T, max_pairs, tables, circuit, msm, total, host_index, host}
void residency_plan(size_t n_g, int fr_bits, size_t fq_bytes, int levels, int c_full, size_t budget, size_t* out) {
  const MsmLayout l = msm_plan_residency(shape_of(n_g, fr_bits, fq_bytes, levels), c_full, std::min(c_full, MSM_REDUCED_WINDOW), MSM_MIN_WINDOW,
                                         budget, 0, 0);
  const size_t v[10] = {(size_t)l.c, (size_t)l.W, (size_t)l.T, l.max_pairs, l.bytes.tables, l.bytes.circuit, l.bytes.msm, l.bytes.total(),
                        l.bytes.host_index ? 1u : 0u, l.bytes.host};
  for (int i = 0; i < 10; i++) out[i] = v[i];
}
// the search of one residency only: out = {c, W, T, max_pairs, total}
void residency_search(size_t n_g, int fr_bits, size_t fq_bytes, int levels, int c_full, size_t budget, int host, size_t* out) {
  const MsmLayout l = msm_plan_layout(shape_of(n_g, fr_bits, fq_bytes, levels), c_full, std::min(c_full, MSM_REDUCED_WINDOW), MSM_MIN_WINDOW,
                                      budget, 0, 0, host != 0);
  const size_t v[5] = {(size_t)l.c, (size_t)l.W, (size_t)l.T, l.max_pairs, l.bytes.total()};
  for (int i = 0; i < 5; i++) out[i] = v[i];
}
// out = {tables, circuit, msm, total, host} for a circuit with |K| = K, |H| = H
void residency_bytes(size_t n_g, int fr_bits, size_t fq_bytes, int levels, int c, int T, size_t max_pairs, size_t K, size_t H, int host,
                     size_t* out) {
  const MsmBytes b = msm_model_bytes(shape_of(n_g, fr_bits, fq_bytes, levels), c, T, max_pairs, K, H, host != 0);
  out[0] = b.tables;
  out[1] = b.circuit;
  out[2] = b.msm;
  out[3] = b.total();
  out[4] = b.host;
}
}
