#include "msm_impl.cuh"
namespace b2m { template struct Msm<FrBls377, FqBls377>; }
