// Curve-independent interface of the device-resident index / prover (Level 2 of include/b2m.h).
#pragma once
#include <string>
#include <vector>

#include "common.cuh"

struct b2m_srs;

namespace b2m {

struct IndexBase {
  virtual ~IndexBase() {}
  // `Marlin::prove` [reference src/lib.rs:151-311]
  virtual void prove(const uint64_t* formatted_input, size_t n_input, const uint64_t* witness, size_t n_witness, b2m_rng* zk_rng,
                     std::vector<uint8_t>& proof) = 0;
  // Copy an instance (x, w) into HBM ahead of time; a later prove() with null pointers uses it.
  virtual void stage(const uint64_t* formatted_input, size_t n_input, const uint64_t* witness, size_t n_witness) = 0;
  // joint non-zeros, |K| and the entries of A, B, C (b2m_index_sizes)
  virtual void sizes(size_t* num_non_zero, size_t* domain_k, size_t* matrix_nnz) const = 0;
  // b2m_index_export
  virtual void export_keys(uint8_t* vectors, uint64_t* const* row_ptrs, uint64_t* const* cols, uint8_t* const* coeffs) = 0;
  int host_resident = 0;            // the twelve |K|-vectors live in pinned host memory (b2m_index_residency)
  size_t host_bytes = 0;            // their pinned bytes
  std::vector<uint8_t> vk_bytes;    // IndexVerifierKey::write (ToBytes)
  std::vector<uint64_t> comms_xy;   // six index commitments, affine Montgomery limbs
  std::string timings_json;
};

IndexBase* make_index_bls(b2m_srs* srs, int pc, size_t num_constraints, size_t num_variables, size_t num_instance,
                          const b2m_matrix* a, const b2m_matrix* b, const b2m_matrix* c);
IndexBase* make_index_bn(b2m_srs* srs, int pc, size_t num_constraints, size_t num_variables, size_t num_instance,
                         const b2m_matrix* a, const b2m_matrix* b, const b2m_matrix* c);
IndexBase* make_index_bls377(b2m_srs* srs, int pc, size_t num_constraints, size_t num_variables, size_t num_instance,
                             const b2m_matrix* a, const b2m_matrix* b, const b2m_matrix* c);

// An index from a key file (b2m_index_load).  bad receives (vector, index, reason) of the first failed check.
IndexBase* load_index_bls(b2m_srs* srs, int pc, size_t num_constraints, size_t num_variables, size_t num_instance, size_t num_non_zero,
                          const b2m_matrix* a, const b2m_matrix* b, const b2m_matrix* c, const uint8_t* const* vectors, const size_t* lens,
                          const uint64_t* comms_xy, bool check_commitments, size_t bad[3]);
IndexBase* load_index_bn(b2m_srs* srs, int pc, size_t num_constraints, size_t num_variables, size_t num_instance, size_t num_non_zero,
                         const b2m_matrix* a, const b2m_matrix* b, const b2m_matrix* c, const uint8_t* const* vectors, const size_t* lens,
                         const uint64_t* comms_xy, bool check_commitments, size_t bad[3]);
IndexBase* load_index_bls377(b2m_srs* srs, int pc, size_t num_constraints, size_t num_variables, size_t num_instance, size_t num_non_zero,
                             const b2m_matrix* a, const b2m_matrix* b, const b2m_matrix* c, const uint8_t* const* vectors, const size_t* lens,
                             const uint64_t* comms_xy, bool check_commitments, size_t bad[3]);

// `PC::commit` over host polynomials (Level 1 of include/b2m.h)
void pc_commit_bls(b2m_srs* srs, int pc, size_t n_polys, const uint64_t* const* coeffs, const size_t* n_coeffs,
                   const int64_t* degree_bounds, const int64_t* hiding_bounds, b2m_rng* rng, uint64_t* out_comm_xy,
                   uint64_t* out_shifted_xy, uint64_t* out_rand, uint64_t* out_shifted_rand, size_t rand_stride);
void pc_commit_bn(b2m_srs* srs, int pc, size_t n_polys, const uint64_t* const* coeffs, const size_t* n_coeffs,
                  const int64_t* degree_bounds, const int64_t* hiding_bounds, b2m_rng* rng, uint64_t* out_comm_xy,
                  uint64_t* out_shifted_xy, uint64_t* out_rand, uint64_t* out_shifted_rand, size_t rand_stride);
void pc_commit_bls377(b2m_srs* srs, int pc, size_t n_polys, const uint64_t* const* coeffs, const size_t* n_coeffs,
                      const int64_t* degree_bounds, const int64_t* hiding_bounds, b2m_rng* rng, uint64_t* out_comm_xy,
                      uint64_t* out_shifted_xy, uint64_t* out_rand, uint64_t* out_shifted_rand, size_t rand_stride);

// `PC::open_combinations` over host polynomials, and `PC::open` as its one-point case (Level 1 of include/b2m.h)
void pc_open_combinations_bls(b2m_srs* srs, int pc, int64_t max_degree_bound, size_t n_polys, const uint64_t* const* coeffs, const size_t* n_coeffs,
                              const int64_t* degree_bounds, const int* hiding, const uint64_t* rands, const uint64_t* shifted_rands, size_t rand_stride,
                              size_t n_lcs, const size_t* lc_term_off, const int64_t* lc_poly, const uint64_t* lc_coeff, size_t n_queries,
                              const size_t* query_lc, const size_t* query_point, size_t n_points, const uint64_t* points,
                              const uint64_t* opening_challenge, uint64_t* out_w_xy, int* out_has_random_v, uint64_t* out_random_v);
void pc_open_combinations_bn(b2m_srs* srs, int pc, int64_t max_degree_bound, size_t n_polys, const uint64_t* const* coeffs, const size_t* n_coeffs,
                             const int64_t* degree_bounds, const int* hiding, const uint64_t* rands, const uint64_t* shifted_rands, size_t rand_stride,
                             size_t n_lcs, const size_t* lc_term_off, const int64_t* lc_poly, const uint64_t* lc_coeff, size_t n_queries,
                             const size_t* query_lc, const size_t* query_point, size_t n_points, const uint64_t* points,
                             const uint64_t* opening_challenge, uint64_t* out_w_xy, int* out_has_random_v, uint64_t* out_random_v);
void pc_open_combinations_bls377(b2m_srs* srs, int pc, int64_t max_degree_bound, size_t n_polys, const uint64_t* const* coeffs,
                                 const size_t* n_coeffs, const int64_t* degree_bounds, const int* hiding, const uint64_t* rands,
                                 const uint64_t* shifted_rands, size_t rand_stride, size_t n_lcs, const size_t* lc_term_off, const int64_t* lc_poly,
                                 const uint64_t* lc_coeff, size_t n_queries, const size_t* query_lc, const size_t* query_point, size_t n_points,
                                 const uint64_t* points, const uint64_t* opening_challenge, uint64_t* out_w_xy, int* out_has_random_v,
                                 uint64_t* out_random_v);

}  // namespace b2m
