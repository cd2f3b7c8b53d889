// Host-side G2 arithmetic for the G2 half of `KZG10::setup` [U ark-poly-commit kzg10::setup]: h, beta * h and the few
// beta^(-e) * h that SonicKZG10's verifier key keeps (`neg_powers_of_h`).  The PROVER never touches G2 (reference
// src/lib.rs:151-311 only commits and opens in G1), so this is a handful of scalar multiplications per key on the CPU with
// the same limb code as the device (field.cuh compiled for the host), written out in ark-serialize's uncompressed form so that
// an SRS file made here can be loaded by arkworks (tools/replay_rs).
//
// Fq2 and the G2 group law live in g2.cuh (shared with the GPU's SRS decoder).
#pragma once
#include <cstdint>
#include <cstring>
#include <vector>

#include "field.cuh"
#include "g2.cuh"

namespace b2m {

// `CanonicalSerialize::serialize_uncompressed` of a short-Weierstrass affine point over Fq2 [U ark-ec 0.3
// short_weierstrass_jacobian.rs + ark-ff QuadExtField]: x.c0 || x.c1 || y.c0 || y.c1, canonical little-endian, with the
// infinity flag (bit 6) in the very last byte; infinity is written as all-zero coordinates + the flag.
template <class Fq>
void g2_write_uncompressed(std::vector<uint8_t>& out, const G2Jac<Fq>& p) {
  const size_t nb = Fq::N * 4;
  if (p.is_inf()) {
    out.insert(out.end(), 4 * nb - 1, 0);
    out.push_back(1u << 6);
    return;
  }
  Fq2<Fq> x, y;
  p.to_affine(&x, &y);
  const Fq* parts[4] = {&x.c0, &x.c1, &y.c0, &y.c1};
  for (const Fq* f : parts) {
    const Fq c = f->to_canonical();
    const uint8_t* b = reinterpret_cast<const uint8_t*>(c.l);
    out.insert(out.end(), b, b + nb);
  }
}

}  // namespace b2m
