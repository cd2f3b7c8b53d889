// Curve-independent interface of the batched verifier (Level 2 of include/b2m.h: b2m_vk_*, b2m_verify*).
#pragma once
#include <string>
#include <vector>

#include "common.cuh"
#include "pc_check.hpp"

struct b2m_srs;

namespace b2m {

struct VerifierBase {
  virtual ~VerifierBase() {}
  // `Marlin::verify` [reference src/lib.rs:315-433] for n proofs, proof i under keys[key_of[i]] (keys of this key's curve and
  // context, repeats allowed); verdicts[i] = 1 / 0 / -1 (malformed).  Every key of the call gets its timings_json.
  virtual void verify_multi(size_t n_keys, VerifierBase* const* keys, size_t n, const uint32_t* key_of, const uint64_t* const* public_inputs,
                            const size_t* n_inputs, const uint8_t* const* proofs, const size_t* proof_lens, b2m_rng* rng, int* verdicts) = 0;
  // n proofs under this key: the one-key case of verify_multi
  void verify_batch(size_t n, const uint64_t* const* public_inputs, const size_t* n_inputs, const uint8_t* const* proofs,
                    const size_t* proof_lens, b2m_rng* rng, int* verdicts) {
    VerifierBase* self = this;
    const std::vector<uint32_t> key_of(n, 0);
    verify_multi(1, &self, n, key_of.data(), public_inputs, n_inputs, proofs, proof_lens, rng, verdicts);
  }
  std::string timings_json;
};

struct VkArgs {
  int pc;
  size_t num_constraints, num_variables, num_non_zero;
  const uint64_t* index_comms_xy;
  const uint64_t* g_xy;
  const uint64_t* gamma_g_xy;
  const uint8_t* h_bytes;
  const uint8_t* beta_h_bytes;
  size_t n_bounds;
  const uint64_t* bounds;
  const void* bound_points;
};

// `PC::VerifierKey` of MarlinKZG10 / SonicKZG10 (Level 1 of include/b2m.h: b2m_pc_vk_*, b2m_pc_check_combinations)
struct PcVkArgs {
  int pc;
  size_t max_degree;
  const uint64_t* g_xy;
  const uint64_t* gamma_g_xy;
  const uint8_t* h_bytes;
  const uint8_t* beta_h_bytes;
  size_t n_bounds;
  const uint64_t* bounds;
  const void* bound_points;
};
struct PcVerifierBase {
  virtual ~PcVerifierBase() {}
  // `PC::check_combinations` for S.n independent sets; verdicts[s] = 1 / 0 / -1 (malformed).  An `Err` of upstream's throws
  // B2M_ERR_INVALID_ARG naming the set before any work or rng draw.
  virtual void check_combinations(const PcSets& S, b2m_rng* rng, int* verdicts) = 0;
  std::string timings_json;
};

// b2m_pairing_check for one curve (pairing_impl.cuh; instantiated with the verifier of that curve)
template <class Fq>
void pairing_check(Ctx& cx, size_t n_g2, const uint8_t* g2, size_t n_products, const size_t* off, const uint64_t* g1_xy, const uint32_t* g2_index,
                   int* verdicts);

// b2m_srs_check_powers for one curve (srs_check_impl.cuh; instantiated with the verifier of that curve)
template <class Fr, class Fq>
void srs_check_powers(b2m_srs* srs, const uint8_t* h, const uint8_t* beta_h, size_t n_neg, const uint64_t* neg_keys, const uint8_t* neg_h,
                      b2m_rng* rng, int* ok, int* bad_kind, size_t* bad_index);

VerifierBase* make_verifier_bls(Ctx& cx, const VkArgs& a);
VerifierBase* make_verifier_bn(Ctx& cx, const VkArgs& a);
VerifierBase* make_verifier_bls377(Ctx& cx, const VkArgs& a);
PcVerifierBase* make_pc_verifier_bls(Ctx& cx, const PcVkArgs& a);
PcVerifierBase* make_pc_verifier_bn(Ctx& cx, const PcVkArgs& a);
PcVerifierBase* make_pc_verifier_bls377(Ctx& cx, const PcVkArgs& a);

}  // namespace b2m
