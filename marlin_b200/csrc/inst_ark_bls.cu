#include "ark_points_impl.cuh"
namespace b2m {
B2M_INSTANTIATE_ARK_POINTS(FqBls)
}  // namespace b2m
