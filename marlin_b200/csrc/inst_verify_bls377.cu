#include "verify_impl.cuh"
namespace b2m {
VerifierBase* make_verifier_bls377(Ctx& cx, const VkArgs& a) { return new MarlinVerifier<FrBls377, FqBls377>(cx, a); }
}  // namespace b2m
