// Batch conversion of ark-serialize G1 / G2 points and Fr elements on the GPU (the SRS and index-key loaders:
// b2m_g1_decode_ark, b2m_g2_decode_ark, b2m_g1_decode_lem, b2m_g2_decode_lem, b2m_g1_to_compressed, b2m_fr_decode_ark, b2m_fr_to_canonical).  Definitions in ark_points_impl.cuh, instantiated per curve by inst_ark_{bls,bn,bls377}.cu.
#pragma once
#include "common.cuh"
#include "field.cuh"

namespace b2m {

// Points are decoded in chunks of this many, so the device scratch stays bounded whatever the input size.
constexpr size_t ARK_DECODE_CHUNK = (size_t)1 << 18;

// The lowest-indexed invalid point of a batch: index == n when every point is valid; reason = a G1_* status (g1_decode.cuh).
struct ArkBad {
  size_t index;
  int reason;
};

// n points in either form -> affine Montgomery limbs (x || y, infinity = 0, 0).  Stops at the first chunk holding an invalid
// point; out_xy is then filled below that chunk only.
template <class Fq>
ArkBad g1_decode_ark(Ctx& cx, const uint8_t* bytes, size_t n, bool compressed, uint64_t* out_xy);
// n points in either form -> uncompressed canonical bytes (4 * sizeof(Fq) each).
template <class Fq>
ArkBad g2_decode_ark(Ctx& cx, const uint8_t* bytes, size_t n, bool compressed, uint8_t* out);
// n snarkjs LEM points (.ptau files; g1_decode.cuh) -> affine Montgomery limbs / uncompressed canonical ark bytes, with the
// same chunking and stopping rule as the ark forms.
template <class Fq>
ArkBad g1_decode_lem_points(Ctx& cx, const uint8_t* bytes, size_t n, uint64_t* out_xy);
template <class Fq>
ArkBad g2_decode_lem_points(Ctx& cx, const uint8_t* bytes, size_t n, uint8_t* out);
// affine Montgomery limbs -> compressed bytes (sizeof(Fq) each).
template <class Fq>
void g1_to_compressed(Ctx& cx, const uint64_t* points_xy, size_t n, uint8_t* out);

// Cause reported by fr_decode_ark for an element that is not below the field modulus.
constexpr int FR_NOT_CANONICAL = 1;

// n canonical little-endian Fr values (sizeof(Fr) bytes each, host memory) -> Montgomery Fr in DEVICE memory out_dev.
// Every chunk is decoded; the lowest index of an element >= r over the whole input is returned (index == n: all valid).
template <class Fr>
ArkBad fr_decode_ark(Ctx& cx, const uint8_t* bytes, size_t n, Fr* out_dev);
// n Montgomery Fr in DEVICE memory -> canonical little-endian bytes in host memory.
template <class Fr>
void fr_to_canonical(Ctx& cx, const Fr* in_dev, size_t n, uint8_t* out);

}  // namespace b2m
