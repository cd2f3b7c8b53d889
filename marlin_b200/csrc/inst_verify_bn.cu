#include "verify_impl.cuh"
namespace b2m {
VerifierBase* make_verifier_bn(Ctx& cx, const VkArgs& a) { return new MarlinVerifier<FrBn, FqBn>(cx, a); }
}  // namespace b2m
