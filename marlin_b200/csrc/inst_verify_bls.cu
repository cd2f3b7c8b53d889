#include "verify_impl.cuh"
namespace b2m {
VerifierBase* make_verifier_bls(Ctx& cx, const VkArgs& a) { return new MarlinVerifier<FrBls, FqBls>(cx, a); }
}  // namespace b2m
