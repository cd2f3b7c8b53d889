#include "prover_impl.cuh"
namespace b2m {
IndexBase* make_index_bls377(b2m_srs* srs, int pc, size_t nc, size_t nv, size_t ni, const b2m_matrix* a, const b2m_matrix* b,
                           const b2m_matrix* c) {
  std::unique_ptr<MarlinIndex<FrBls377, FqBls377>> idx(new MarlinIndex<FrBls377, FqBls377>(srs, srs->ctx->ntt_bls377(), *srs->bls377, pc, nc, nv, ni));
  idx->build(a, b, c);
  return idx.release();
}
IndexBase* load_index_bls377(b2m_srs* srs, int pc, size_t nc, size_t nv, size_t ni, size_t nnz, const b2m_matrix* a, const b2m_matrix* b,
                          const b2m_matrix* c, const uint8_t* const* vectors, const size_t* lens, const uint64_t* comms_xy, bool check_commitments,
                          size_t bad[3]) {
  using I = MarlinIndex<FrBls377, FqBls377>;
  std::unique_ptr<I> idx(new I(srs, srs->ctx->ntt_bls377(), *srs->bls377, pc, nc, nv, ni));
  typename I::LoadBad lb{0, 0, 0};
  try {
    idx->load(a, b, c, nnz, vectors, lens, comms_xy, check_commitments, &lb);
  } catch (...) {
    bad[0] = lb.vector; bad[1] = lb.index; bad[2] = (size_t)lb.reason;
    throw;
  }
  return idx.release();
}
void pc_commit_bls377(b2m_srs* srs, int pc, size_t n_polys, const uint64_t* const* coeffs, const size_t* n_coeffs,
                   const int64_t* degree_bounds, const int64_t* hiding_bounds, b2m_rng* rng, uint64_t* out_comm_xy, uint64_t* out_shifted_xy,
                   uint64_t* out_rand, uint64_t* out_shifted_rand, size_t rand_stride) {
  pc_commit_impl<FrBls377, FqBls377>(srs, *srs->bls377, pc, n_polys, coeffs, n_coeffs, degree_bounds, hiding_bounds, rng, out_comm_xy, out_shifted_xy, out_rand,
                             out_shifted_rand, rand_stride);
}
void pc_open_combinations_bls377(b2m_srs* srs, int pc, int64_t max_degree_bound, size_t n_polys, const uint64_t* const* coeffs, const size_t* n_coeffs,
                              const int64_t* degree_bounds, const int* hiding, const uint64_t* rands, const uint64_t* shifted_rands, size_t rand_stride,
                              size_t n_lcs, const size_t* lc_term_off, const int64_t* lc_poly, const uint64_t* lc_coeff, size_t n_queries,
                              const size_t* query_lc, const size_t* query_point, size_t n_points, const uint64_t* points,
                              const uint64_t* opening_challenge, uint64_t* out_w_xy, int* out_has_random_v, uint64_t* out_random_v) {
  pc_open_combinations_impl<FrBls377, FqBls377>(srs, *srs->bls377, pc, max_degree_bound, n_polys, coeffs, n_coeffs, degree_bounds, hiding, rands, shifted_rands,
                                        rand_stride, n_lcs, lc_term_off, lc_poly, lc_coeff, n_queries, query_lc, query_point, n_points, points,
                                        opening_challenge, out_w_xy, out_has_random_v, out_random_v);
}
}  // namespace b2m
