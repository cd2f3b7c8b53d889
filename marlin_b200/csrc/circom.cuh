// circom constraint systems on the GPU (b2m_circom_decode_constraints) and the satisfiability check of any padded R1CS
// (b2m_r1cs_check).  Definitions in circom_impl.cuh, instantiated per curve by inst_circom_{bls,bn,bls377}.cu.
#pragma once
#include "common.cuh"
#include "field.cuh"

namespace b2m {

// Bytes of one constraint-section term: u32 wire id, then a 32-byte canonical coefficient (n8 = 32) [U circom r1csfile].
constexpr size_t CIRCOM_TERM_BYTES = 36;

// The lowest bad term of a constraint section, in file order: matrix 0/1/2 = A/B/C, term = its index in that matrix's
// term array (row_ptrs[matrix]), reason 1 = wire >= nWires, 2 = coefficient not below r (0: every term is valid).
struct CircomBad {
  int matrix;
  size_t term;
  int reason;
};

// m constraints of a `.r1cs` section 2 (host bytes, len of them) whose term-count prefix sums b2m_circom_constraint_rows
// wrote -> three CSR matrices in row normal form (columns ascending, duplicate wires summed, zeros dropped), Montgomery
// coefficients, wire w at column w (w < ni0) or w + shift.  out_row_ptr[j] holds m + 1 entries; out_col[j] / out_coeff[j]
// hold at least row_ptrs[j][m] entries (normalising never adds one).  Chunks of whole constraints run in file order and
// the first chunk holding a bad term stops the call.
template <class Fr>
CircomBad circom_decode_constraints(Ctx& cx, const uint8_t* bytes, size_t len, size_t m, const uint64_t* const* row_ptrs, uint64_t n_wires,
                                    uint64_t ni0, uint64_t shift, uint64_t* const* out_row_ptr, uint64_t* const* out_col, uint64_t* const* out_coeff);

// ark-relations' `which_is_unsatisfied` on a padded R1CS in `b2m_matrix` form: the lowest row r with
// <A_r, z> * <B_r, z> != <C_r, z>, z = instance || witness (Montgomery), or nc when every row holds.
template <class Fr>
size_t r1cs_check(Ctx& cx, size_t nc, size_t nv, size_t ni, const b2m_matrix* const* mats, const uint64_t* instance, const uint64_t* witness);

}  // namespace b2m
