#include "ark_points_impl.cuh"
namespace b2m {
B2M_INSTANTIATE_ARK_POINTS(FqBls)
B2M_INSTANTIATE_ARK_FR(FrBls)
}  // namespace b2m
