// b2m_srs_check_powers: is a device-resident key one chain of powers of a secret beta?  (DESIGN.md "Powers-of-Tau files")
//
// Relations, numbered in one list in this order (P_i = powers_of_g[i], G_k = the gamma power of key k, N_k = beta^-k h):
//   family 0   e(P_{i+1}, h) = e(P_i, beta h)          i = 0 .. D - 1
//   family 1   e(G_{k+1}, h) = e(G_k, beta h)          consecutive keys k, k + 1 both held, k ascending
//   family 2   e(P_k, N_k)   = e(P_0, h)               every neg key, in the caller's order
//   family 3   e(G_k, N_k)   = e(G_0, h)               every neg key whose G_k is held, in the caller's order
// A check of a range [a, b) of that list draws one independent 128-bit randomiser per relation and folds the range into
//   e(A, h) * e(-B, beta h) * e(E, h) * prod_k e(C_k, N_k) = 1,
//   A = sum_i r_i P_{i+1} + sum_k s_k G_{k+1},  B = sum_i r_i P_i + sum_k s_k G_k,
//   C_k = t_k P_k + u_k G_k,  E = -(sum t_k) P_0 - (sum u_k) G_0.
// A and B are two MSMs over the slices [a + 1, b + 1) and [a, b) of the window tables with the same device-resident scalars
// r_i, the gamma terms riding as the blinding group; E and the C_k are one-pair MSMs (+ one gamma term).  If every relation
// holds the product is 1; if one fails, the product is 1 for at most one value of its randomiser given the others
// (verify_impl.cuh, DESIGN.md §9), so a bad range passes with probability at most 2^-128.
//
// Randomisers: a check takes two next_u64() per relation, family 0 first (ascending i), then families 1-3 in list order.  A
// ChaCha rng's family-0 words are generated on the device at the stream position (srs_check_rand_kernel), a callback rng is
// drawn on the host and uploaded; both read the same words in the same order.  A failing range is split in halves, both
// checked in one level (MSM batch + one pairing launch) with fresh randomisers, left before right, and the search follows the
// lower failing half: the result is the lowest failing relation, so that of the first failing family.
#pragma once
#include <algorithm>
#include <vector>

#include "capi_types.cuh"
#include "hostutil.hpp"
#include "pairing_impl.cuh"
#include "poly_impl.cuh"  // chacha_block_dev, ChaChaKey

namespace b2m {

// out[j] = stream words [pos0 + 4j, pos0 + 4j + 4) as a canonical 128-bit Fr: the j-th pair of next_u64() draws
template <class Fr>
__global__ void srs_check_rand_kernel(ChaChaKey key, int rounds, uint64_t pos0, size_t n, Fr* out) {
  const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j >= n) return;
  const uint64_t pos = pos0 + 4ull * j;
  uint32_t w[32];
  chacha_block_dev(key.k, pos >> 4, rounds, w);
  const int off = (int)(pos & 15);
  if (off + 4 > 16) chacha_block_dev(key.k, (pos >> 4) + 1, rounds, w + 16);
  Fr v = Fr::zero();
#pragma unroll
  for (int k = 0; k < 4; k++) v.l[k] = w[off + k];
  st_fr(out + j, v);
}

template <class Fr, class Fq>
struct SrsPowerCheck {
  using Pt = Affine<Fq>;
  Ctx& cx;
  b2m_srs* srs;
  Msm<Fr, Fq>& msm;
  size_t D, n_gamma;
  std::vector<uint64_t> f1_key;               // family 1: the lower key k
  std::vector<size_t> f1_lo, f1_hi;           // ... slots of G_k and G_{k+1}
  std::vector<uint64_t> neg_key;              // family 2: neg key per relation (its N is G2 point 2 + index)
  std::vector<size_t> f3_neg, f3_slot;        // family 3: neg-key index and slot of G_k
  size_t gamma0_slot = SIZE_MAX;              // slot of G_0 (families 3 need it)
  std::unique_ptr<PairingG2Set<Fq>> g2;       // h, beta h, N_0 .. N_{n_neg - 1}
  ZkSource<b2m_rng> zr;
  int checks = 0;

  static Fr fr_u128(uint64_t lo, uint64_t hi) {
    Fr c = Fr::zero();
    c.l[0] = (uint32_t)lo; c.l[1] = (uint32_t)(lo >> 32); c.l[2] = (uint32_t)hi; c.l[3] = (uint32_t)(hi >> 32);
    return Fr::from_canonical(c);
  }

  SrsPowerCheck(b2m_srs* s, const uint8_t* h, const uint8_t* beta_h, size_t n_neg, const uint64_t* neg_keys, const uint8_t* neg_h, b2m_rng* rng)
      : cx(s->ctx->cx), srs(s), msm(*s->msm<Fr>()), D(s->n_g - 1), n_gamma(s->n_gamma), zr(rng) {
    constexpr size_t G2B = 4 * Fq::N * 4;
    auto finite = [&](const uint8_t* p) { return !((p[G2B - 1] >> 6) & 1u); };
    B2M_REQUIRE(finite(h) && finite(beta_h), B2M_ERR_INVALID_ARG, "h / beta_h is the point at infinity");
    std::vector<std::pair<uint64_t, size_t>> keys;  // (key, slot), sorted
    for (size_t k = 0; k < n_gamma; k++) keys.push_back({srs->gamma_idx[k], k});
    std::sort(keys.begin(), keys.end());
    for (size_t k = 0; k + 1 < keys.size(); k++)
      if (keys[k + 1].first == keys[k].first + 1) {
        f1_key.push_back(keys[k].first);
        f1_lo.push_back(keys[k].second);
        f1_hi.push_back(keys[k + 1].second);
      }
    for (const auto& kv : keys)
      if (kv.first == 0) gamma0_slot = kv.second;
    for (size_t j = 0; j < n_neg; j++) {
      B2M_REQUIRE(neg_keys[j] <= D, B2M_ERR_INVALID_ARG, "neg key %llu is above the max degree %zu", (unsigned long long)neg_keys[j], D);
      B2M_REQUIRE(finite(neg_h + j * G2B), B2M_ERR_INVALID_ARG, "neg_h[%zu] is the point at infinity", j);
      neg_key.push_back(neg_keys[j]);
      if (gamma0_slot == SIZE_MAX) continue;
      for (const auto& kv : keys)
        if (kv.first == neg_keys[j]) {
          f3_neg.push_back(j);
          f3_slot.push_back(kv.second);
        }
    }
    std::vector<uint8_t> g2b(h, h + G2B);
    g2b.insert(g2b.end(), beta_h, beta_h + G2B);
    if (n_neg) g2b.insert(g2b.end(), neg_h, neg_h + n_neg * G2B);
    g2.reset(new PairingG2Set<Fq>(cx, 2 + n_neg, g2b.data()));
  }

  size_t relations() const { return D + f1_key.size() + neg_key.size() + f3_neg.size(); }
  // relation -> (family, i or k)
  std::pair<int, size_t> name(size_t r) const {
    if (r < D) return {0, r};
    r -= D;
    if (r < f1_key.size()) return {1, (size_t)f1_key[r]};
    r -= f1_key.size();
    if (r < neg_key.size()) return {2, (size_t)neg_key[r]};
    return {3, (size_t)neg_key[f3_neg[r - neg_key.size()]]};
  }

  // one level: pass[n] = whether range nodes[n] passed its check
  std::vector<int> check(const std::vector<std::pair<size_t, size_t>>& nodes, const char* span) {
    const size_t sp_msm = cx.span_begin(span, (double)nodes.size());
    // family-0 randomisers of every node, in node order, on the device
    size_t n0 = 0;
    for (const auto& nd : nodes) n0 += std::min(nd.second, D) - std::min(nd.first, D);
    DBuf<Fr> dr(cx, std::max<size_t>(n0, 1));
    std::vector<Fr> small(1, Fr::zero());  // canonical: [0] = zero, then every job's one-pair scalar and gamma vector
    struct Job {
      bool dev;
      size_t off, n, base_off, g_off, n2;
    };
    std::vector<Job> jobs;
    struct Pair {
      size_t job;
      uint32_t g2;
      bool neg;
    };
    std::vector<std::vector<Pair>> prods;
    size_t at0 = 0;
    const size_t F1 = D + f1_key.size(), F2 = F1 + neg_key.size();
    for (const auto& nd : nodes) {
      const size_t a0 = std::min(nd.first, D), len0 = std::min(nd.second, D) - a0;
      if (len0) {
        if (!zr.callback) {
          ChaChaKey key;
          memcpy(key.k, zr.cc.key, sizeof(key.k));
          srs_check_rand_kernel<Fr><<<div_up(len0, 256), 256, 0, cx.stream>>>(key, zr.cc.rounds, zr.cc.word_pos, len0, dr.p + at0);
          B2M_CHECK_LAUNCH();
          cx.launches++;
          zr.cc.word_pos += 4ull * len0;
        } else {
          std::vector<Fr> hr(len0);
          for (Fr& v : hr) {
            const uint64_t lo = zr.next_u64(), hi = zr.next_u64();
            v = fr_u128(lo, hi).to_canonical();
          }
          B2M_CUDA(cudaMemcpyAsync(dr.p + at0, hr.data(), len0 * sizeof(Fr), cudaMemcpyHostToDevice, cx.stream));
          cx.sync();
        }
      }
      // gamma vectors of A and B, E's scalars, the C_k
      auto gvec = [&]() {
        const size_t g = small.size();
        small.resize(small.size() + n_gamma, Fr::zero());
        return g;
      };
      const size_t gA = gvec(), gB = gvec();
      std::vector<Fr> ga(n_gamma, Fr::zero()), gb(n_gamma, Fr::zero());
      Fr e_p0 = Fr::zero(), e_g0 = Fr::zero();
      std::vector<std::pair<size_t, std::pair<Fr, Fr>>> cs;  // neg index -> (t, u)
      auto c_of = [&](size_t j) -> std::pair<Fr, Fr>& {
        for (auto& c : cs)
          if (c.first == j) return c.second;
        cs.push_back({j, {Fr::zero(), Fr::zero()}});
        return cs.back().second;
      };
      for (size_t r = std::max(nd.first, D); r < nd.second; r++) {
        const uint64_t lo = zr.next_u64(), hi = zr.next_u64();
        const Fr x = fr_u128(lo, hi);
        if (r < F1) {
          ga[f1_hi[r - D]] = ga[f1_hi[r - D]] + x;
          gb[f1_lo[r - D]] = gb[f1_lo[r - D]] + x;
        } else if (r < F2) {
          c_of(r - F1).first = x;
          e_p0 = e_p0 - x;
        } else {
          const size_t q = r - F2;
          c_of(f3_neg[q]).second = x;
          e_g0 = e_g0 - x;
        }
      }
      for (size_t k = 0; k < n_gamma; k++) {
        small[gA + k] = ga[k].to_canonical();
        small[gB + k] = gb[k].to_canonical();
      }
      std::vector<Pair> pr;
      const size_t jA = jobs.size();
      jobs.push_back(len0 ? Job{true, at0, len0, a0 + 1, gA, n_gamma} : Job{false, 0, 1, 0, gA, n_gamma});
      jobs.push_back(len0 ? Job{true, at0, len0, a0, gB, n_gamma} : Job{false, 0, 1, 0, gB, n_gamma});
      pr.push_back(Pair{jA, 0, false});
      pr.push_back(Pair{jA + 1, 1, true});
      if (!cs.empty()) {
        const size_t s = small.size();
        small.push_back(e_p0.to_canonical());
        const size_t g = gvec();
        if (gamma0_slot != SIZE_MAX) small[g + gamma0_slot] = e_g0.to_canonical();
        jobs.push_back(Job{false, s, 1, 0, g, n_gamma});
        pr.push_back(Pair{jobs.size() - 1, 0, false});
        for (const auto& c : cs) {
          const size_t sc = small.size();
          small.push_back(c.second.first.to_canonical());
          const size_t gc = gvec();
          for (size_t q = 0; q < f3_neg.size(); q++)
            if (f3_neg[q] == c.first) small[gc + f3_slot[q]] = c.second.second.to_canonical();
          jobs.push_back(Job{false, sc, 1, (size_t)neg_key[c.first], gc, n_gamma});
          pr.push_back(Pair{jobs.size() - 1, (uint32_t)(2 + c.first), false});
        }
      }
      prods.push_back(pr);
      at0 += len0;
    }
    DBuf<Fr> ds(cx, small.size());
    ds.upload(small.data(), small.size());
    DBuf<Pt> dres(cx, jobs.size());
    for (size_t j0 = 0; j0 < jobs.size(); j0 += MSM_MAX_BATCH) {
      MsmJob<Fr, Fq> mj[MSM_MAX_BATCH];
      const int m = (int)std::min<size_t>(MSM_MAX_BATCH, jobs.size() - j0);
      for (int k = 0; k < m; k++) {
        const Job& jb = jobs[j0 + k];
        mj[k] = MsmJob<Fr, Fq>{(jb.dev ? dr.p : ds.p) + jb.off, false, jb.n, jb.base_off, jb.n2 ? ds.p + jb.g_off : nullptr, jb.n2, 0, nullptr, 0,
                               nullptr, dres.p + j0 + k};
      }
      msm.run_batch(mj, m);
    }
    std::vector<Pt> res(jobs.size());
    dres.download(res.data(), jobs.size());
    cx.sync();
    cx.span_end(sp_msm);
    std::vector<Pt> g1;
    std::vector<uint32_t> g2i;
    std::vector<size_t> off{0};
    for (const auto& pr : prods) {
      for (const Pair& p : pr) {
        const Pt& q = res[p.job];
        g1.push_back(p.neg ? Pt{q.x, q.y.neg()} : q);
        g2i.push_back(p.g2);
      }
      off.push_back(g1.size());
    }
    std::vector<int> ok(prods.size());
    const size_t sp_pair = cx.span_begin("srs_check_pairing", (double)prods.size());
    g2->check(prods.size(), off.data(), reinterpret_cast<const uint64_t*>(g1.data()), g2i.data(), ok.data());
    cx.span_end(sp_pair);
    checks += (int)nodes.size();
    return ok;
  }

  // ok = 1, or ok = 0 with the lowest failing relation
  void run(int* ok, int* bad_kind, size_t* bad_index) {
    const size_t R = relations();
    *ok = 1;
    if (check({{0, R}}, "srs_check_msm")[0] != 1) {
      std::pair<size_t, size_t> node{0, R};
      while (node.second - node.first > 1) {
        const size_t mid = node.first + (node.second - node.first) / 2;
        const std::vector<int> v = check({{node.first, mid}, {mid, node.second}}, "srs_check_bisection");
        if (v[0] != 1) node = {node.first, mid};
        else if (v[1] != 1) node = {mid, node.second};
        // both halves passed: a bad relation met a 2^-128 event; the node is checked again with fresh randomisers
      }
      const auto nm = name(node.first);
      *ok = 0;
      if (bad_kind) *bad_kind = nm.first;
      if (bad_index) *bad_index = nm.second;
    }
    zr.commit_position();
  }
};

template <class Fr, class Fq>
void srs_check_powers(b2m_srs* srs, const uint8_t* h, const uint8_t* beta_h, size_t n_neg, const uint64_t* neg_keys, const uint8_t* neg_h,
                      b2m_rng* rng, int* ok, int* bad_kind, size_t* bad_index) {
  SrsPowerCheck<Fr, Fq>(srs, h, beta_h, n_neg, neg_keys, neg_h, rng).run(ok, bad_kind, bad_index);
}

}  // namespace b2m
