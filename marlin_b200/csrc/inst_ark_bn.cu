#include "ark_points_impl.cuh"
namespace b2m {
B2M_INSTANTIATE_ARK_POINTS(FqBn)
}  // namespace b2m
