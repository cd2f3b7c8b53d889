#include "ntt_impl.cuh"
namespace b2m { template struct Ntt<FrBls377>; }
