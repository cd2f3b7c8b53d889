// Host build of marlin_b200/csrc/msm_layout.hpp -- the MSM key layout planner and its byte model -- for
// tests/test_msm_tables_host.py.
#include "../../marlin_b200/csrc/msm_layout.hpp"

using namespace b2m;

static MsmKeyShape shape_of(size_t n_g, size_t n_extra, int fr_bits, size_t fq_bytes, int levels) {
  MsmKeyShape k;
  k.n_g = n_g;
  k.n_extra = n_extra;
  k.fr_bits = fr_bits;
  k.fq_bytes = fq_bytes;
  k.affine_levels = levels;
  return k;
}

extern "C" {
// out = {c, W, T, max_pairs, tables, circuit, msm, total}
void layout_plan(size_t n_g, size_t n_extra, int fr_bits, size_t fq_bytes, int levels, int c_full, int c_reduced, int c_min, size_t budget,
                 int forced_T, size_t forced_cap, size_t* out) {
  const MsmLayout l = msm_plan_layout(shape_of(n_g, n_extra, fr_bits, fq_bytes, levels), c_full, c_reduced, c_min, budget, forced_T, forced_cap);
  const size_t v[8] = {(size_t)l.c, (size_t)l.W, (size_t)l.T, l.max_pairs, l.bytes.tables, l.bytes.circuit, l.bytes.msm, l.bytes.total()};
  for (int i = 0; i < 8; i++) out[i] = v[i];
}
// out = {tables, circuit, msm, total} for the largest circuit of the key
void layout_bytes(size_t n_g, size_t n_extra, int fr_bits, size_t fq_bytes, int levels, int c, int T, size_t max_pairs, size_t* out) {
  const MsmBytes b = msm_model_bytes_largest(shape_of(n_g, n_extra, fr_bits, fq_bytes, levels), c, T, max_pairs);
  out[0] = b.tables;
  out[1] = b.circuit;
  out[2] = b.msm;
  out[3] = b.total();
}
int layout_sets_fit(int c, int m) { return msm_sets_fit(c, m) ? 1 : 0; }
}
