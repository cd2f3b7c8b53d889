#include "circom_impl.cuh"
namespace b2m {
B2M_INSTANTIATE_CIRCOM(FrBn)
}  // namespace b2m
