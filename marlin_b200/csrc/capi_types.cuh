// Definitions of the opaque handles of include/b2m.h and the host-buffer wrappers of Level 0.
#pragma once
#include <cstdio>
#include <memory>
#include <string>
#include <type_traits>

#include "common.cuh"
#include "msm.cuh"
#include "ntt.cuh"

namespace b2m {
extern thread_local std::string g_last_error;

template <class F>
int guard(F&& f) {
  try {
    f();
    return B2M_OK;
  } catch (const Error& e) {
    g_last_error = e.what();
    return e.code;
  } catch (const std::exception& e) {
    g_last_error = e.what();
    return B2M_ERR_INVALID_ARG;
  }
}
}  // namespace b2m

// Lifetimes: an index / committer key borrows its SRS, an SRS borrows its context.  Destroying a parent while children are
// alive only marks it; the storage goes when the last child is destroyed, so no destroy order is a use-after-free.
struct b2m_ctx {
  b2m::Ctx cx;
  int children = 0;
  bool dead = false;
  std::unique_ptr<b2m::Ntt<b2m::FrBls>> ntt_bls_;
  std::unique_ptr<b2m::Ntt<b2m::FrBn>> ntt_bn_;
  std::unique_ptr<b2m::Ntt<b2m::FrBls377>> ntt_bls377_;
  explicit b2m_ctx(int device) : cx(device) {}
  b2m::Ntt<b2m::FrBls>& ntt_bls() {
    if (!ntt_bls_) ntt_bls_.reset(new b2m::Ntt<b2m::FrBls>(cx));
    return *ntt_bls_;
  }
  b2m::Ntt<b2m::FrBn>& ntt_bn() {
    if (!ntt_bn_) ntt_bn_.reset(new b2m::Ntt<b2m::FrBn>(cx));
    return *ntt_bn_;
  }
  b2m::Ntt<b2m::FrBls377>& ntt_bls377() {
    if (!ntt_bls377_) ntt_bls377_.reset(new b2m::Ntt<b2m::FrBls377>(cx));
    return *ntt_bls377_;
  }
  template <class Fr>
  b2m::Ntt<Fr>& ntt() {
    if constexpr (std::is_same<Fr, b2m::FrBls>::value) return ntt_bls();
    else if constexpr (std::is_same<Fr, b2m::FrBn>::value) return ntt_bn();
    else return ntt_bls377();
  }
};

namespace b2m {
template <class Fr_, class Fq_>
struct CurveTypes {
  using Fr = Fr_;
  using Fq = Fq_;
};
// f(CurveTypes<Fr, Fq>{}) for a curve id (B2M_CURVE_*); an unknown id is B2M_ERR_INVALID_ARG
template <class F>
auto with_curve(int curve, F&& f) {
  switch (curve) {
    case B2M_CURVE_BLS12_381: return f(CurveTypes<FrBls, FqBls>{});
    case B2M_CURVE_BN254: return f(CurveTypes<FrBn, FqBn>{});
    case B2M_CURVE_BLS12_377: return f(CurveTypes<FrBls377, FqBls377>{});
  }
  throw Error(B2M_ERR_INVALID_ARG, "unknown curve id");
}
// B2M_ERR_INVALID_ARG unless curve is a known curve id
inline void require_curve(int curve) {
  with_curve(curve, [](auto) {});
}
}  // namespace b2m

struct b2m_srs {
  b2m_ctx* ctx;
  int children = 0;
  bool dead = false;
  int curve;
  size_t n_g, n_gamma;
  std::unique_ptr<b2m::Msm<b2m::FrBls, b2m::FqBls>> bls;
  std::unique_ptr<b2m::Msm<b2m::FrBn, b2m::FqBn>> bn;
  std::unique_ptr<b2m::Msm<b2m::FrBls377, b2m::FqBls377>> bls377;
  // gamma_idx[k] = the power of beta held in slot k of the powers_of_gamma_g (they live in the window
  // tables right after the G1 powers: see Msm::n_extra)
  std::vector<uint64_t> gamma_idx;

  // slot of beta^i * gamma * G, or throws
  size_t gamma_slot(uint64_t i) const {
    for (size_t k = 0; k < gamma_idx.size(); k++)
      if (gamma_idx[k] == i) return k;
    throw b2m::Error(B2M_ERR_INVALID_ARG, b2m::fmt("the SRS holds no power %llu of gamma*G", (unsigned long long)i));
  }

  b2m::MsmKeyShape shape;   // what the byte model knows of this key
  b2m::MsmLayout layout;    // the planned layout and the model's figures for it
  size_t budget = 0;        // pool bytes available when the key was created

  // the key's MSM (std::unique_ptr) of the curve whose scalar field is Fr
  template <class Fr>
  auto& msm() {
    if constexpr (std::is_same<Fr, b2m::FrBls>::value) return bls;
    else if constexpr (std::is_same<Fr, b2m::FrBn>::value) return bn;
    else return bls377;
  }

  b2m_srs(b2m_ctx* c, int curve_, const uint64_t* g, size_t ng, const uint64_t* gamma, const uint64_t* gidx, size_t ngamma,
          int window_bits, int window_tables)
      : ctx(c), curve(curve_), n_g(ng), n_gamma(ngamma) {
    using namespace b2m;
    for (size_t k = 0; k < ngamma; k++) gamma_idx.push_back(gidx ? gidx[k] : k);
    with_curve(curve, [&](auto t) {
      using Fr = typename decltype(t)::Fr;
      using Fq = typename decltype(t)::Fq;
      plan<Fr, Fq>(window_bits, window_tables);
      msm<Fr>().reset(new Msm<Fr, Fq>(c->cx, reinterpret_cast<const Affine<Fq>*>(g), ng, reinterpret_cast<const Affine<Fq>*>(gamma), ngamma,
                                      layout.c, false, layout.T, layout.max_pairs));
    });
    c->cx.sync();
  }

  // Layout of the key (msm_layout.hpp): all W window tables whenever the byte model of the largest circuit the key can index
  // fits min(free device memory, the context's memory limit); else the largest T < W and MSM pass cap that fit; only when no
  // layout fits with a device-resident index, the same search with a host-resident one (layout.bytes.host_index); else
  // B2M_ERR_MEMORY_LIMIT before anything is allocated.  window_tables > 0 (or B2M_MSM_TABLES) forces T, B2M_MSM_MAX_PAIRS the
  // pass cap (tests).  A multi-GPU context keeps its tables sharded by rank instead: the full layout only.
  template <class Fr, class Fq>
  void plan(int window_bits, int window_tables) {
    using namespace b2m;
    Ctx& cx = ctx->cx;
    int forced_T = window_tables;
    size_t forced_cap = 0;
    if (const char* e = getenv("B2M_MSM_TABLES")) forced_T = atoi(e);
    if (const char* e = getenv("B2M_MSM_MAX_PAIRS")) forced_cap = (size_t)atoll(e);
    B2M_REQUIRE(window_bits == 0 || (window_bits >= MSM_MIN_WINDOW && window_bits <= 24), B2M_ERR_INVALID_ARG, "window bits %d out of range [%d, 24]",
                window_bits, MSM_MIN_WINDOW);
    B2M_REQUIRE(n_g >= 1, B2M_ERR_INVALID_ARG, "SRS size %zu out of range", n_g);
    shape = MsmKeyShape{n_g, n_gamma, Fr::Params::BITS, sizeof(Fq), Fq::N > 8 ? 3 : 0};
    if (const char* e = getenv("B2M_MSM_AFFINE_LEVELS")) shape.affine_levels = atoi(e);
    const int c_full = window_bits > 0 ? window_bits : Msm<Fr, Fq>::pick_window(n_g / (size_t)(cx.world > 1 ? cx.world : 1));
    if (cx.world > 1) {  // (Msm rejects a forced reduction with B2M_ERR_UNSUPPORTED)
      layout.c = c_full;
      layout.T = forced_T;
      layout.max_pairs = forced_cap;
      return;
    }
    const int c_reduced = window_bits > 0 ? window_bits : std::min(c_full, MSM_REDUCED_WINDOW);
    const int c_min = window_bits > 0 ? window_bits : MSM_MIN_WINDOW;
    if (forced_T > 0 && forced_T < msm_windows(shape.fr_bits, c_full)) {  // a forced T the bucket field cannot hold is a bad argument
      bool fits = false;
      for (int c = c_reduced; c >= c_min && !fits; c--) fits = msm_sets_fit(c, msm_sets(msm_windows(shape.fr_bits, c), forced_T));
      const int m = msm_sets(msm_windows(shape.fr_bits, c_reduced), forced_T);
      B2M_REQUIRE(fits, B2M_ERR_INVALID_ARG, "%d window table(s) at c = %d need %d bucket sets of 2^%d buckets, more than the 2^%d bucket ids",
                  forced_T, c_reduced, m, c_reduced - 1, MSM_BKT_BITS);
    }
    budget = cx.memory_budget();
    layout = msm_plan_residency(shape, c_full, c_reduced, c_min, budget, forced_T, forced_cap);
    const MsmBytes& b = layout.bytes;
    B2M_REQUIRE(layout.T > 0, B2M_ERR_MEMORY_LIMIT,
                "an SRS of %zu powers needs %zu bytes (window tables %zu, index and prover %zu, MSM scratch %zu at %d table(s), c = %d, "
                "%zu-pair passes) for the largest circuit it can index; the device-memory budget is %zu bytes",
                n_g, b.total(), b.tables, b.circuit, b.msm, layout.T ? layout.T : 1, layout.c, layout.max_pairs, budget);
  }

  // Residency of an index of |K| = K, |H| = H on this key, before it allocates (true: the twelve |K|-vectors go to pinned host
  // memory once the index is built).  Device residency whenever the model of its index, prover and MSM scratch (sized for this
  // circuit's largest MSM, not the whole key) fits what the budget leaves; otherwise host residency if that model fits.  With
  // a memory limit set and neither fitting, B2M_ERR_MEMORY_LIMIT naming both (without a limit the device-resident index is
  // tried, as it always was).  force_host (B2M_INDEX_HOST, tests) takes host residency whatever fits.  Host residency is
  // refused when MemAvailable (/proc/meminfo) is below the bytes it pins, and on multi-GPU contexts.  held: bytes the index
  // already took for structures the model's index term counts (its matrices), added back to the budget.
  bool require_fits(size_t K, size_t H, bool force_host, size_t held) const {
    using namespace b2m;
    Ctx& cx = ctx->cx;
    if (cx.world > 1) {
      B2M_REQUIRE(!force_host, B2M_ERR_UNSUPPORTED, "a host-resident index needs a single-GPU context (this one is rank %d of %d)", cx.rank, cx.world);
      return false;
    }
    const MsmBytes d = msm_model_bytes(shape, layout.c, layout.T, layout.max_pairs, K, H, false);
    const MsmBytes h = msm_model_bytes(shape, layout.c, layout.T, layout.max_pairs, K, H, true);
    bool host = force_host;
    const size_t avail = cx.memory_budget() + held;
    if (!host && d.circuit + d.msm > avail) {
      host = h.circuit + h.msm <= avail;
      B2M_REQUIRE(host || !cx.memory_limit, B2M_ERR_MEMORY_LIMIT,
                  "an index of |K| = %zu, |H| = %zu needs %zu bytes device-resident (index and prover %zu, MSM scratch %zu) or %zu bytes "
                  "host-resident (index and prover %zu, %zu bytes pinned on the host); the device-memory budget leaves %zu bytes",
                  K, H, d.circuit + d.msm, d.circuit, d.msm, h.circuit + h.msm, h.circuit, h.host, avail);
    }
    if (host && cx.memory_limit)
      B2M_REQUIRE(h.circuit + h.msm <= avail, B2M_ERR_MEMORY_LIMIT,
                  "a host-resident index of |K| = %zu, |H| = %zu needs %zu bytes (index and prover %zu, MSM scratch %zu); the device-memory "
                  "budget leaves %zu bytes", K, H, h.circuit + h.msm, h.circuit, h.msm, avail);
    if (host) {
      const size_t mem = host_mem_available();
      B2M_REQUIRE(h.host <= mem, B2M_ERR_MEMORY_LIMIT, "a host-resident index of |K| = %zu pins %zu bytes of host memory; MemAvailable is %zu bytes", K,
                  h.host, mem);
    }
    return host;
  }
  // MemAvailable of /proc/meminfo in bytes (SIZE_MAX when it cannot be read)
  static size_t host_mem_available() {
    FILE* f = fopen("/proc/meminfo", "r");
    if (!f) return (size_t)-1;
    char line[256];
    size_t kb = (size_t)-1;
    while (fgets(line, sizeof line, f)) {
      unsigned long long v = 0;
      if (sscanf(line, "MemAvailable: %llu kB", &v) == 1) {
        kb = (size_t)v;
        break;
      }
    }
    fclose(f);
    return kb == (size_t)-1 ? kb : kb * 1024;
  }
  template <class G>
  auto with_msm(G&& g) const {
    if (bls) return g(*bls);
    if (bn) return g(*bn);
    return g(*bls377);
  }
  int window_bits() const { return with_msm([](const auto& m) { return m.c; }); }
  int window_tables() const { return with_msm([](const auto& m) { return m.T; }); }
  int affine_levels() const { return with_msm([](const auto& m) { return m.affine_levels; }); }
  size_t affine_min_refs() const { return with_msm([](const auto& m) { return m.affine_min_refs; }); }
};


// `PC::CommitterKey` after `PC::trim`: a validated view of the device-resident SRS
struct b2m_ck {
  b2m_srs* srs;
  int pc;
  size_t supported_degree, hiding_bound;
  std::vector<uint64_t> bounds;  // enforced degree bounds, sorted
  int64_t max_bound() const { return bounds.empty() ? -1 : (int64_t)bounds.back(); }
  bool enforced(uint64_t b) const {
    for (uint64_t x : bounds)
      if (x == b) return true;
    return false;
  }
};

void b2m_release_ctx(b2m_ctx* ctx);
void b2m_release_srs(b2m_srs* srs);
