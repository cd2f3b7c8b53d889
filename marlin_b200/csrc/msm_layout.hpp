// Device-memory layout of an MSM key -- how many window tables it keeps and how many pairs one bucket pass takes -- and the
// byte model that chooses it.  Host-only C++ (no CUDA): capi_types.cuh plans every single-GPU SRS with it, and
// tests/host/msm_layout_host_shim.cpp compiles it on its own.
//
// A key keeps T <= W window tables.  With m = ceil(W / T) table j holds 2^(c m j) P_i, and window w reads table w / m and
// sends its digit to bucket set w % m; the sets are reduced separately and recombined as sum_k 2^(c k) S_k (Horner).  T = W
// (m = 1) is the full layout: one bucket set, no recombination.
#pragma once
#include <algorithm>
#include <cstddef>
#include <cstdint>

namespace b2m {

constexpr int MSM_MIN_WINDOW = 8;  // at most ceil(256 / 8) = 32 windows
constexpr int MSM_BKT_BITS = 24;   // a sorted reference is {table index | sign << 31, bucket | table << 24}
constexpr int MSM_MAX_BATCH = 8;   // MSMs per run_batch call
constexpr size_t MSM_AFFINE_MIN_REFS = (size_t)1 << 23;  // MSMs with fewer bucket references skip the batched-affine levels (latency-bound below)
// Window width of a key that cannot keep all its tables: the bucket array grows to m 2^(c-1) points per MSM of a batch, which
// at c = 20 and m = 13 is 10.5 GB for a batch of 8 (BLS12-381); c = 16 keeps it at 0.8 GB even at T = 1 (m = 16).
constexpr int MSM_REDUCED_WINDOW = 16;
// Pass caps the planner tries, largest first (after "no cap"); the smallest is the floor of the model.
constexpr int MSM_PASS_LOG_MAX = 22, MSM_PASS_LOG_MIN = 16;

inline int msm_windows(int fr_bits, int c) { return (fr_bits + 1 + c - 1) / c; }
inline int msm_sets(int W, int T) { return (W + T - 1) / T; }
// Tables the kernels read with m = msm_sets(W, T) sets: windows w < W use tables w / m < ceil(W / m).  A requested T is
// normalised to this (T = 15 at W = 16 gives m = 2, which reads 8 tables), so no table is built that no MSM reads.
inline int msm_tables_used(int W, int T) { return (W + msm_sets(W, T) - 1) / msm_sets(W, T); }
// bucket ids k * 2^(c-1) + (|d| - 1) of all m sets fit the 24-bit bucket field of a sorted reference
inline bool msm_sets_fit(int c, int m) { return ((size_t)m << (c - 1)) <= ((size_t)1 << MSM_BKT_BITS); }

// What the byte model needs to know about a key and its curve.
struct MsmKeyShape {
  size_t n_g = 0;         // G1 powers
  size_t n_extra = 0;     // gamma powers stored after them in every table
  int fr_bits = 255;      // Fr::Params::BITS
  size_t fq_bytes = 48;   // sizeof(Fq)
  int affine_levels = 3;  // Msm::affine_levels
};

// The pool hands out blocks in its own granularity, so the bytes it counts in use exceed the bytes asked for by up to a
// block per live allocation; a key's plan keeps this much room for that (an index check, made after the key's own
// allocations, does not count it again).
constexpr size_t MSM_POOL_SLACK = (size_t)256 << 20;

struct MsmBytes {
  size_t tables = 0;   // the T window tables
  size_t circuit = 0;  // index structures plus the larger of the index-build temporaries and the prover's buffers
  size_t msm = 0;      // scratch of one run_batch call of MSM_MAX_BATCH jobs, each pass as large as the cap allows
  bool host_index = false;  // the circuit term keeps the twelve |K|-vectors of the index in pinned host memory
  size_t host = 0;          // pinned host bytes of a host-resident index (not part of total())
  size_t total() const { return tables + circuit + msm + MSM_POOL_SLACK; }
};

// A host-resident index streams its vectors to the prover in chunks of this many Fr, two device slots per streamed vector
// (round 3 streams at most three vectors at once).
constexpr size_t INDEX_STREAM_CHUNK = (size_t)1 << 20;
constexpr int INDEX_STREAM_VECS = 3;

// Largest circuit a key of n_g powers can index: |K| - 1 <= D and 3 |H| - 1 <= D (D = n_g - 1, AHP max degree, zk bound 1).
inline size_t msm_pow2_floor(size_t x) {
  size_t p = 1;
  while (p * 2 <= x) p *= 2;
  return p;
}
inline size_t msm_largest_k(size_t n_g) { return msm_pow2_floor(n_g ? n_g : 1); }
inline size_t msm_largest_h(size_t n_g) { return msm_pow2_floor(n_g / 3 ? n_g / 3 : 1); }

// The largest MSM of a circuit: no committed polynomial has more than max(3|H|, |K|) coefficients (the AHP max degree + 1,
// zk bound 1), and none has more than the key's n_g.
inline size_t msm_largest_pairs(size_t n_g, size_t K, size_t H) { return std::min(n_g, std::max(K, 3 * H)); }

// THE byte model: an upper bound on the stream-ordered pool bytes that a key of layout (c, T, max_pairs) holds together with
// the index and one proof of a circuit with |K| = K, |H| = H, at the peak of `index` or `prove`.  Written from the allocation
// sites; every term names them.  host_index: the index keeps its twelve |K|-vectors in pinned host memory once it is built.
inline MsmBytes msm_model_bytes(const MsmKeyShape& k, int c, int T, size_t max_pairs, size_t K, size_t H, bool host_index = false) {
  const size_t fr = 32, aff = 2 * k.fq_bytes, xyzz = 4 * k.fq_bytes;
  const int W = msm_windows(k.fr_bits, c), m = msm_sets(W, T);
  T = msm_tables_used(W, T);
  MsmBytes b;
  b.tables = (size_t)T * (k.n_g + k.n_extra) * aff;  // Msm::tables
  // prover_impl.cuh.  Resident index: ieval / ipoly (12 K Fr, `vecs`), the CSR of A and B (each matrix has at most K entries),
  // the column buckets of A, B, C for t(X), the NTT twiddles (half of the largest domain, max(2K, 4H)).
  const size_t vecs = 12 * K * fr;
  const size_t index = 2 * (4 * (H + 1) + K * (4 + fr)) + 4 * (H + 1) + 3 * K * (4 + 1 + fr) + std::max(K, 2 * H) * fr;
  // Index build (5 nnz vectors of the joint matrix, the work and evaluation vectors; load: the evaluation and NTT work
  // vectors), always with the twelve vectors on the device.
  const size_t build = 3 * K * (8 + 3 * fr) + 2 * K * fr;
  // One proof, the largest of its phases (in units of Fr; every vector of |H| or |H| + 1 counted as H + 1):
  //  * alive from rounds 1-2 to the end: the staged and the proof's z, z_A, z_B, x(X), w(X), z_A(X), z_B(X), the 3|H| mask,
  //    the 4|H| `summed` evaluations, r(alpha, X) evaluations and coefficients, t(X), z(X), g_1, the 2|H| h_1: 22 (H + 1);
  //  * rounds 1-2: the four 4|H| vectors of q_1 and fft_padded's 4|H| work vector: 20 (H + 1) more (round 1's mask sampling,
  //    t(X)'s 3|K| products and the 4|H| evaluations of z_A, z_B are freed before them and smaller: 5H, 3K + H and 12H);
  //  * round 3: f, h_2; b, f evaluations and b(X); the three 2|K| vectors of b f and fft_padded's 2|K| work vector: 13 K;
  //  * the opening: the evaluations' suffix vectors of g_1, g_2 and z_b / t (2 (H + 1) + K), and per point the combination,
  //    its suffix sums and at most the merged witness scalars (4 n; n = 3|H| at beta, |K| at gamma), besides f and h_2.
  const size_t live = 22 * (H + 1);
  const size_t r12 = live + 20 * (H + 1);
  const size_t r3 = live + 13 * K;
  const size_t open = live + 2 * (H + 1) + 3 * K + 12 * (H + 1) + 4 * K;
  const size_t prove = std::max(std::max(r12, r3), open) * fr;
  // A host-resident index at rest holds no |K|-vector; round 3 and the opening stream them through the stager's slots.
  const size_t stager = 2 * (size_t)INDEX_STREAM_VECS * std::min(K, INDEX_STREAM_CHUNK) * fr;
  if (host_index) {
    b.circuit = std::max(index + vecs + build, index + prove + stager);
    b.host_index = true;
    b.host = vecs;
  } else {
    b.circuit = index + vecs + std::max(build, prove);
  }
  // msm_impl.cuh run_batch: the circuit's largest MSM (plus a few blinding pairs), or one pass of max_pairs pairs.
  const size_t nb = (size_t)m << (c - 1);  // buckets per MSM
  const size_t largest = msm_largest_pairs(k.n_g, K, H);
  const size_t pairs = (max_pairs && max_pairs < largest ? max_pairs : largest) + 64;
  const size_t refs = (size_t)W * pairs;
  const size_t threads = refs / 32 + 256 + 1;
  size_t s = 2 * refs * (4 + 8);                          // digits + sorted, two slots
  s += 2 * 3 * 4 * (nb + 1);                              // hist, offsets, cursor, two slots
  s += 2 * threads * (4 + xyzz);                          // part_bkt + part_pt
  s += 2 * ((size_t)1 << 18) * 16 + (4 * threads / 256 + 4) * (16 + xyzz);  // long / short runs, final runs + chunk_pt
  if (k.affine_levels > 0 && refs >= MSM_AFFINE_MIN_REFS) {  // batched-affine level buffers
    size_t bound[8] = {refs};
    const int LV = std::min(k.affine_levels, 6);
    for (int l = 1; l <= LV; l++) bound[l] = (bound[l - 1] + nb) / 2 + 1;
    const size_t slots = 64 * ((bound[1] + 63) / 64 + 128);
    s += bound[1] * aff + (LV > 1 ? bound[2] * aff : 0) + bound[LV] * 8 + 3 * 4 * (nb + 1) + slots * (16 + k.fq_bytes) + (slots + 256) * k.fq_bytes;
  }
  s += (size_t)MSM_MAX_BATCH * nb * xyzz;                 // buckets
  s += (size_t)MSM_MAX_BATCH * m * ((nb / m) / 4 + 8192) * xyzz;  // row / column partials and sums of the reduction
  s += (size_t)MSM_MAX_BATCH * (m + (largest / (max_pairs ? max_pairs : largest) + 1)) * xyzz;  // set sums, pass sums
  b.msm = s;
  return b;
}
inline MsmBytes msm_model_bytes_largest(const MsmKeyShape& k, int c, int T, size_t max_pairs, bool host_index = false) {
  return msm_model_bytes(k, c, T, max_pairs, msm_largest_k(k.n_g), msm_largest_h(k.n_g), host_index);
}

struct MsmLayout {
  int c = 0, W = 0, T = 0;  // window bits, windows, window tables kept (T = 0: nothing fits)
  size_t max_pairs = 0;     // pairs per MSM pass (0: no cap)
  MsmBytes bytes;           // the model's figures for this layout
};

// Layout of a single-GPU key under a budget of pool bytes: all W tables at the key's own window width c_full whenever the
// model fits (with no pass cap if that fits, else the largest cap that does); only otherwise c_reduced and the largest T
// below the full W at the widest window in [c_min, c_reduced] that fits, again with the largest cap that fits.  Only
// T = ceil(W / m) are considered (msm_tables_used): any other T has the sets of the next such T and idle tables.  forced_T /
// forced_cap (> 0) fix those choices (forced_T >= W: the full layout; other T normalised); c_min = c_reduced = c_full fixes
// the window.  When nothing fits, T = 0 and `bytes` holds the smallest layout's figures.  host_index: the circuit term of a
// host-resident index (msm_model_bytes).
inline MsmLayout msm_plan_layout(const MsmKeyShape& k, int c_full, int c_reduced, int c_min, size_t budget, int forced_T, size_t forced_cap,
                                 bool host_index = false) {
  MsmLayout best;
  auto caps_try = [&](int c, int T, MsmLayout& out) {
    for (int lg = MSM_PASS_LOG_MAX + 1; lg >= MSM_PASS_LOG_MIN; lg--) {
      size_t cap = lg > MSM_PASS_LOG_MAX ? 0 : (size_t)1 << lg;
      if (forced_cap) {
        if (lg != MSM_PASS_LOG_MAX + 1) break;
        cap = forced_cap;
      } else if (cap && cap >= k.n_g) {
        continue;  // no cap
      }
      const MsmBytes b = msm_model_bytes_largest(k, c, T, cap, host_index);
      out = MsmLayout{c, msm_windows(k.fr_bits, c), T, cap, b};
      if (b.total() <= budget) return true;
    }
    return false;
  };
  const int W_full = msm_windows(k.fr_bits, c_full);
  if (forced_T <= 0 || forced_T >= W_full) {
    if (caps_try(c_full, W_full, best)) return best;
    if (forced_T >= W_full) {
      best.T = 0;
      return best;
    }
  }
  // A reduced layout keeps fewer tables than the full one (so T, and the table bytes, only grow with the budget).  For each
  // T the widest window from c_reduced down that fits is taken: on a small key the m 2^(c-1) buckets of a batch, not the
  // tables, are what a narrower window saves.
  for (int T = forced_T > 0 ? forced_T : W_full - 1; T >= 1; T--) {
    for (int c = c_reduced; c >= c_min; c--) {
      const int W = msm_windows(k.fr_bits, c);
      if (T > W || !msm_sets_fit(c, msm_sets(W, T))) continue;
      const int Tu = msm_tables_used(W, T);
      if (forced_T <= 0 && Tu != T) continue;  // (reached again as T = Tu)
      if (caps_try(c, Tu, best)) return best;
    }
    if (forced_T > 0) break;
  }
  best.T = 0;
  return best;
}

// Residency rule: exactly the device-resident search first (every T and pass cap); only when nothing fits, the same search
// with the index's twelve |K|-vectors in pinned host memory.  The result's bytes.host_index records which one planned it;
// when neither fits, T = 0 and `bytes` holds the device search's smallest layout.  (So the tables kept are monotone in the
// budget within each residency, not across the switch: a host-resident plan may keep more tables than the device-resident
// plan of a slightly larger budget.)
inline MsmLayout msm_plan_residency(const MsmKeyShape& k, int c_full, int c_reduced, int c_min, size_t budget, int forced_T, size_t forced_cap) {
  const MsmLayout dev = msm_plan_layout(k, c_full, c_reduced, c_min, budget, forced_T, forced_cap, false);
  if (dev.T > 0) return dev;
  const MsmLayout host = msm_plan_layout(k, c_full, c_reduced, c_min, budget, forced_T, forced_cap, true);
  return host.T > 0 ? host : dev;
}

}  // namespace b2m
