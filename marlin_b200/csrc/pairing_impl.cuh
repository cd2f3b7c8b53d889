// The GPU pairing product check behind b2m_pairing_check and the batched verifier's checks: one thread per product runs the
// Miller loop over its pairs and the final exponentiation of pairing.cuh.  G2 line coefficients are computed on the host once
// per distinct G2 point (a handful per call) and read by every thread from global memory: threads of a warp at the same step of
// products over the same G2 point read the same words.
#pragma once
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "devmem.cuh"
#include "pairing.cuh"

namespace b2m {

// bounds of one launch: at most PAIRING_PRODUCT_CHUNK products and max(PAIRING_PAIR_CHUNK, pairs of the largest product)
// pairs, so device scratch stays bounded by that whatever the caller passes
constexpr size_t PAIRING_PRODUCT_CHUNK = (size_t)1 << 16, PAIRING_PAIR_CHUNK = (size_t)1 << 18;

template <class Fq>
__global__ void __launch_bounds__(64) pairing_check_kernel(size_t n, const uint32_t* off, const Affine<Fq>* g1, const uint32_t* g2_index,
                                                             const G2Line<Fq>* lines, const uint8_t* g2_inf, const PairingConsts<Fq> C,
                                                             int* verdicts, unsigned long long* first_bad) {
  constexpr int NL = ate_line_count<Fq>();
  const size_t k = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint32_t a = off[k], m = off[k + 1] - a;
  for (uint32_t j = 0; j < m; j++)
    if (!g1_pairing_input_ok(ld_words(g1 + a + j))) {
      atomicMin(first_bad, (unsigned long long)(a + j));
      verdicts[k] = -1;
      return;
    }
  const Fq12T<Fq> f = miller_loop_ate<Fq>(
      (int)m, [&](int j) { return ld_words(g1 + a + j); },
      [&](int j) -> const G2Line<Fq>* {
        const uint32_t q = g2_index[a + j];
        return g2_inf[q] ? nullptr : lines + (size_t)q * NL;
      });
  verdicts[k] = final_exponentiation_ate(f, C).is_one() ? 1 : 0;
}

// A set of G2 points, prepared once: their line coefficients on the device.
template <class Fq>
struct PairingG2Set {
  static constexpr int NL = ate_line_count<Fq>();
  Ctx& cx;
  size_t n;
  PairingConsts<Fq> C;
  DBuf<G2Line<Fq>> lines;
  DBuf<uint8_t> inf;

  // bytes: n ark-serialize uncompressed G2 points.  B2M_ERR_SERIALIZATION naming the first one that is non-canonical or off
  // the twist (no subgroup test: see b2m_pairing_check).
  PairingG2Set(Ctx& c, size_t count, const uint8_t* bytes) : cx(c), n(count), C(pairing_consts<Fq>()) {
    std::vector<G2Line<Fq>> h(std::max<size_t>(1, n) * NL);
    std::vector<uint8_t> hinf(std::max<size_t>(1, n), 1);
    for (size_t i = 0; i < n; i++) {
      Fq2<Fq> x, y;
      bool is_inf;
      const int st = g2_affine_uncompressed<Fq>(bytes + i * 4 * Fq::N * 4, &x, &y, &is_inf);
      if (st != G1_OK) throw Error(B2M_ERR_SERIALIZATION, fmt("G2 point %zu: %s", i, point_status_name(st)));
      hinf[i] = is_inf;
      if (!is_inf) g2_lines<Fq>(x, y, C, h.data() + i * NL);
    }
    lines = DBuf<G2Line<Fq>>(cx, h.size());
    inf = DBuf<uint8_t>(cx, hinf.size());
    lines.upload(h.data(), h.size());
    inf.upload(hinf.data(), hinf.size());
  }

  // points of sets prepared before: point i is point src[i].second of set *src[i].first, its lines copied on the device (runs of
  // consecutive points of one set in one copy) rather than computed again
  PairingG2Set(Ctx& c, const std::vector<std::pair<const PairingG2Set*, size_t>>& src) : cx(c), n(src.size()), C(src.at(0).first->C) {
    lines = DBuf<G2Line<Fq>>(cx, n * NL);
    inf = DBuf<uint8_t>(cx, n);
    for (size_t i = 0, j; i < n; i = j) {
      const PairingG2Set* s = src[i].first;
      const size_t q = src[i].second;
      for (j = i + 1; j < n && src[j].first == s && src[j].second == q + (j - i);) j++;
      B2M_CUDA(cudaMemcpyAsync(lines.p + i * NL, s->lines.p + q * NL, (j - i) * NL * sizeof(G2Line<Fq>), cudaMemcpyDeviceToDevice, cx.stream));
      B2M_CUDA(cudaMemcpyAsync(inf.p + i, s->inf.p + q, j - i, cudaMemcpyDeviceToDevice, cx.stream));
    }
  }

  // verdicts[k] = (product k == 1), product k being the pairs [off[k], off[k + 1]) of (g1_xy[j], G2 point g2_index[j]).
  // B2M_ERR_INVALID_ARG for malformed offsets or indices and, naming the pair, for a G1 point off the curve.
  void check(size_t n_products, const size_t* off, const uint64_t* g1_xy, const uint32_t* g2_index, int* verdicts) {
    if (n_products == 0) return;
    for (size_t k = 0; k < n_products; k++)
      B2M_REQUIRE(off[k] <= off[k + 1], B2M_ERR_INVALID_ARG, "product_off is not non-decreasing at %zu", k);
    for (size_t j = off[0]; j < off[n_products]; j++)
      B2M_REQUIRE(g2_index[j] < n, B2M_ERR_INVALID_ARG, "g2_index[%zu] = %u is not below n_g2 = %zu", j, g2_index[j], n);
    const Affine<Fq>* pts = reinterpret_cast<const Affine<Fq>*>(g1_xy);
    size_t max_pairs = 0;
    for (size_t k = 0; k < n_products; k++) max_pairs = std::max(max_pairs, off[k + 1] - off[k]);
    const size_t pair_cap = std::max(PAIRING_PAIR_CHUNK, max_pairs), prod_cap = std::min(n_products, PAIRING_PRODUCT_CHUNK);
    B2M_REQUIRE(pair_cap < ((size_t)1 << 32), B2M_ERR_INVALID_ARG, "a product of %zu pairs", max_pairs);
    DBuf<uint32_t> doff(cx, prod_cap + 1), dindex(cx, std::min(pair_cap, off[n_products] - off[0]) + 1);
    DBuf<Affine<Fq>> dg1(cx, dindex.n);
    DBuf<int> dver(cx, prod_cap);
    DBuf<unsigned long long> dbad(cx, 1);
    std::vector<uint32_t> hoff(prod_cap + 1);
    for (size_t k0 = 0; k0 < n_products;) {
      size_t k1 = k0 + 1;
      while (k1 < n_products && k1 - k0 < prod_cap && off[k1 + 1] - off[k0] <= pair_cap) k1++;
      const size_t m = k1 - k0, p0 = off[k0], np = off[k1] - p0;
      for (size_t k = 0; k <= m; k++) hoff[k] = (uint32_t)(off[k0 + k] - p0);
      B2M_CUDA(cudaMemsetAsync(dbad.p, 0xff, sizeof(unsigned long long), cx.stream));
      doff.upload(hoff.data(), m + 1);
      if (np) {
        dindex.upload(g2_index + p0, np);
        dg1.upload(pts + p0, np);
      }
      const size_t sp = cx.span_begin("pairing_check", (double)m);
      pairing_check_kernel<Fq><<<div_up(m, 64), 64, 0, cx.stream>>>(m, doff.p, dg1.p, dindex.p, lines.p, inf.p, C, dver.p, dbad.p);
      B2M_CHECK_LAUNCH();
      cx.launches++;
      cx.span_end(sp);
      unsigned long long bad = 0;
      dbad.download(&bad, 1);
      dver.download(verdicts + k0, m);
      cx.sync();
      if (bad != ~0ull) throw Error(B2M_ERR_INVALID_ARG, fmt("G1 point %zu is not on the curve (or its limbs are not below p)", p0 + bad));
      k0 = k1;
    }
  }
};

template <class Fq>
void pairing_check(Ctx& cx, size_t n_g2, const uint8_t* g2, size_t n_products, const size_t* off, const uint64_t* g1_xy, const uint32_t* g2_index,
                   int* verdicts) {
  PairingG2Set<Fq> set(cx, n_g2, g2);
  set.check(n_products, off, g1_xy, g2_index, verdicts);
}

}  // namespace b2m
