#include "circom_impl.cuh"
namespace b2m {
B2M_INSTANTIATE_CIRCOM(FrBls377)
}  // namespace b2m
