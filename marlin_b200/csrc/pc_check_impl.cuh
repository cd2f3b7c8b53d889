// Batched Level-1 `PC::check_combinations` for MarlinKZG10 / SonicKZG10 (b2m_pc_check_combinations) over independent opening
// sets, on the Marlin verifier's machinery (verify_impl.cuh):
//   1. validate (host)     upstream's `Err` cases for every set (pc_set_error), before any work or rng draw
//   2. decode (GPU)        every set's commitments, shifted commitments and w's, one thread per point (g1_decode_kernel)
//   3. terms (host)        per set and opening point, the (Fr, base) terms of its pairing equation (pc_check.hpp)
//   4. + 5.                VerifyItems::resolve, an item being a set: one 128-bit randomiser per (set, point) per check, one
//                          G2 group (h, beta h and SonicKZG10's slot per bound), bisection of failing sets (DESIGN.md §16)
#pragma once
#include "verify_impl.cuh"

namespace b2m {

template <class Fr, class Fq>
struct PcVerifier : PcVerifierBase {
  using Pt = Affine<Fq>;
  using Clock = std::chrono::steady_clock;
  static constexpr size_t FQ_BYTES = Fq::N * 4;

  Ctx& cx;
  int pc;
  std::vector<uint64_t> bounds;
  std::vector<Pt> shared;                   // PC_S_*: g, gamma g, MarlinKZG10 shift powers
  std::vector<uint8_t> g2_bytes;            // h, beta h, SonicKZG10's beta^-(D - d) h per bound
  std::unique_ptr<PairingG2Set<Fq>> g2set;  // the same, prepared

  PcVerifier(Ctx& c, const PcVkArgs& a) : cx(c), pc(a.pc), bounds(a.bounds, a.bounds + a.n_bounds) {
    for (size_t k = 0; k < a.n_bounds; k++) {
      B2M_REQUIRE(bounds[k] <= a.max_degree, B2M_ERR_INVALID_ARG, "degree bound %llu exceeds the max degree %zu", (unsigned long long)bounds[k],
                  a.max_degree);
      for (size_t j = 0; j < k; j++) B2M_REQUIRE(bounds[j] != bounds[k], B2M_ERR_INVALID_ARG, "degree bound %llu repeats", (unsigned long long)bounds[k]);
    }
    Pt g, gamma_g;
    memcpy(&g, a.g_xy, sizeof(Pt));
    memcpy(&gamma_g, a.gamma_g_xy, sizeof(Pt));
    shared = {g, gamma_g};
    pc_key_g2<Fq>(cx, pc, a.h_bytes, a.beta_h_bytes, a.n_bounds, a.bound_points, shared, g2_bytes, g2set);
  }

  void check_combinations(const PcSets& S, b2m_rng* rng, int* verdicts) override {
    const Clock::time_point t_all = Clock::now();
    for (size_t s = 0; s < S.n; s++) {
      const std::string e = pc_set_error<Fr>(S, s, bounds);
      B2M_REQUIRE(e.empty(), B2M_ERR_INVALID_ARG, "set %zu: %s", s, e.c_str());
    }
    ZkSource<b2m_rng> zr(rng);
    const size_t NS = shared.size();
    // 2. decode every set's points behind the shared bases
    Clock::time_point t0 = Clock::now();
    std::vector<uint8_t> bytes;
    std::vector<uint32_t> first(S.n);
    std::vector<size_t> count(S.n);
    size_t n_pts = 0;
    for (size_t s = 0; s < S.n; s++) {
      const std::vector<const uint8_t*> p = pc_set_points(pc, S, s, FQ_BYTES);
      for (const uint8_t* b : p) bytes.insert(bytes.end(), b, b + FQ_BYTES);
      first[s] = (uint32_t)(NS + n_pts);
      count[s] = p.size();
      n_pts += p.size();
    }
    DBuf<Pt> bases(cx, NS + n_pts);
    std::vector<int> status;
    bases.upload(shared.data(), NS);
    decode_g1_bases<Fq>(cx, bytes, n_pts, bases.p + NS, status, nullptr);
    const double ms_decode = std::chrono::duration<double, std::milli>(Clock::now() - t0).count();
    // 3. terms
    t0 = Clock::now();
    std::vector<VerifyEq<Fr>> all(S.n);
    for (size_t s = 0; s < S.n; s++) {
      verdicts[s] = 0;
      for (size_t k = 0; k < count[s]; k++)
        if (status[first[s] - NS + k] != G1_OK) verdicts[s] = -1;
    }
    host_parallel(S.n, [&](size_t s) {
      if (verdicts[s] == 0 && !pc_set_equations<Fr>(pc, S, s, bounds, first[s], all[s])) verdicts[s] = -1;
    });
    VerifyItems<Fr, Fq> items(cx);
    items.shared = shared;
    std::vector<size_t> set_of;
    for (size_t s = 0; s < S.n; s++) {
      if (verdicts[s] < 0) continue;
      set_of.push_back(s);
      items.eqs.push_back(std::move(all[s]));
      items.key.push_back(0);
      items.pt_lo.push_back(first[s] - NS);
      items.pt_hi.push_back(first[s] - NS + count[s]);
    }
    const double ms_terms = std::chrono::duration<double, std::milli>(Clock::now() - t0).count();
    // 4. + 5. with this key's G2 points as the call's one group
    const G2Layout L = g2_layout({{g2_bytes.data(), g2_bytes.size() / (4 * FQ_BYTES)}}, 4 * FQ_BYTES);
    double ms_g2 = 0, ms_tables = 0, ms_checks = 0;
    if (!items.eqs.empty()) {
      t0 = Clock::now();
      std::vector<std::pair<const PairingG2Set<Fq>*, size_t>> src;
      for (const auto& p : L.src) src.push_back({g2set.get(), p.second});
      PairingG2Set<Fq> g2(cx, src);
      ms_g2 = std::chrono::duration<double, std::milli>(Clock::now() - t0).count();
      t0 = Clock::now();
      items.msm.reset(new Msm<Fr, Fq>(cx, bases.p + NS, n_pts, shared.data(), NS, 0, true));
      ms_tables = std::chrono::duration<double, std::milli>(Clock::now() - t0).count();
      t0 = Clock::now();
      items.resolve(L, g2, set_of, zr, verdicts);
      ms_checks = std::chrono::duration<double, std::milli>(Clock::now() - t0).count();
    }
    zr.commit_position();
    // terms_ms: step 3; fold_ms: the randomised scalar fold of every check (host), inside first_check_ms + bisection_ms
    timings_json = fmt(
        "{\"sets\": %zu, \"points\": %zu, \"decode_ms\": %.4f, \"terms_ms\": %.4f, \"g2_set_ms\": %.4f, \"msm_tables_ms\": %.4f, "
        "\"fold_ms\": %.4f, \"msm_ms\": %.4f, \"pairing_ms\": %.4f, \"first_check_ms\": %.4f, \"bisection_ms\": %.4f, \"checks\": %d, "
        "\"products\": %d, \"total_ms\": %.4f}",
        S.n, n_pts, ms_decode, ms_terms, ms_g2, ms_tables, items.ms_fold, items.ms_msm, items.ms_pairing, items.ms_first,
        ms_checks - items.ms_first, items.checks, items.products, std::chrono::duration<double, std::milli>(Clock::now() - t_all).count());
  }
};

}  // namespace b2m
