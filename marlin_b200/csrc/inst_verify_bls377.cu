#include "verify_impl.cuh"
#include "pc_check_impl.cuh"
#include "srs_check_impl.cuh"
namespace b2m {
VerifierBase* make_verifier_bls377(Ctx& cx, const VkArgs& a) { return new MarlinVerifier<FrBls377, FqBls377>(cx, a); }
PcVerifierBase* make_pc_verifier_bls377(Ctx& cx, const PcVkArgs& a) { return new PcVerifier<FrBls377, FqBls377>(cx, a); }
template void pairing_check<FqBls377>(Ctx&, size_t, const uint8_t*, size_t, const size_t*, const uint64_t*, const uint32_t*, int*);
template void srs_check_powers<FrBls377, FqBls377>(b2m_srs*, const uint8_t*, const uint8_t*, size_t, const uint64_t*, const uint8_t*, b2m_rng*, int*, int*,
                                             size_t*);
}  // namespace b2m
