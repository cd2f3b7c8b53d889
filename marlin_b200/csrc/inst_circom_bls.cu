#include "circom_impl.cuh"
namespace b2m {
B2M_INSTANTIATE_CIRCOM(FrBls)
}  // namespace b2m
