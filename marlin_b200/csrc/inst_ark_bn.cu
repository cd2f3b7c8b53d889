#include "ark_points_impl.cuh"
namespace b2m {
B2M_INSTANTIATE_ARK_POINTS(FqBn)
B2M_INSTANTIATE_ARK_FR(FrBn)
}  // namespace b2m
