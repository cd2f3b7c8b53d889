#include "ark_points_impl.cuh"
namespace b2m {
B2M_INSTANTIATE_ARK_POINTS(FqBls377)
B2M_INSTANTIATE_ARK_FR(FrBls377)
}  // namespace b2m
