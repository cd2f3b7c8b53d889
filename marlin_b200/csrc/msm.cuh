// Variable-base multi-scalar multiplication over G1 for sm_90a.
//
// Replaces ark-ec 0.3 `VariableBaseMSM::multi_scalar_mul(&[G::Affine], &[BigInt])`
// [U ark-ec src/msm/variable_base.rs] behind `KZG10::commit` / `KZG10::open`, i.e. behind every
// `PC::commit` and `PC::open_combinations` of the prover [R src/lib.rs:172,193,213,292].
//
// The reference runs Pippenger with ~17 windows of c = ln(n)+2 bits, one rayon task per
// window, 2^c-1 Jacobian buckets each, a running-sum reduction per window and c doublings
// between windows.  This design trades HBM capacity for all of the doublings and all but
// one of the bucket sets: the bases are the FIXED powers of the SRS, so at key-load time we
// store 2^(c*w) * P_i for every window w (W tables, W*96 B per power; 5.2 GB for 2^22 powers
// at c = 20).  An MSM is then ONE bucket problem: every (scalar, window) signed digit d sends
// table[w][i] (negated if d < 0) to bucket |d|, and the answer is sum_b b * B_b.
//   1. digits:      Montgomery scalar -> canonical -> W signed c-bit digits, histogram
//   2. scan:        exclusive prefix sum of the 2^(c-1) bucket sizes
//   3. scatter:     counting-sort the (window, index, sign) references by bucket
//   3a. levels:     (381-bit curve, large MSMs) three levels of pairwise BATCHED-AFFINE additions inside every bucket
//                   (msm_affine.cuh): 6 multiplications per addition instead of 10, 7/8 of all additions
//   4. accumulate:  balanced XYZZ mixed additions over what is left (every thread the same number of references),
//                   cut buckets stitched afterwards
//   5. reduce:      sum_b (b+1) B_b through row / column sums of the 2-D bucket view, bit planes, one Horner fold
// The result is a unique group element, compared with the oracle in affine form.
#pragma once
// A key that cannot hold all W tables keeps T < W of them and splits its bucket problem into m = ceil(W / T) bucket sets, and
// long MSMs can run as several bucket passes of at most max_pairs pairs (msm_layout.hpp).
#include "common.cuh"
#include "curve.cuh"
#include "msm_layout.hpp"

namespace b2m {

constexpr uint32_t MSM_BKT_MASK = (1u << MSM_BKT_BITS) - 1;
constexpr uint32_t MSM_NO_DIGIT = 0xffffffffu;
constexpr int MSM_MAX_AFFINE_LEVELS = 6;

template <class Fr, class Fq>
struct MsmJob {
  const Fr* scalars;       // device array
  bool mont;               // Montgomery form (polynomial coefficients) or canonical integers
  size_t n;
  size_t base_off;         // slice powers_of_g[base_off .. base_off + n)
  const Fr* scalars2;      // second scalar group (blinding coefficients) against the extra bases, or null
  size_t n2;
  size_t extra_base;       // first extra base (slot among the powers_of_gamma_g) used by scalars2
  const XYZZ<Fq>* extra;   // further device-resident terms added to the result
  int n_extra;
  XYZZ<Fq>* out_xyzz;      // either output may be null
  Affine<Fq>* out_affine;
  size_t scalar_stride = 1;  // scalars[i * scalar_stride] pairs with powers[base_off + i] (multi-GPU: the rank's residue class)
};

template <class Fr, class Fq>
struct Msm {
  Ctx* ctx;
  size_t n_srs = 0;    // G1 powers resident on THIS GPU (multi-GPU: the powers i = rank mod world, slot i / world)
  size_t n_srs_global = 0;  // powers of the whole key
  int tab_rank = 0, tab_world = 1;  // the communicator layout the tables were built for
  size_t n_extra = 0;  // further fixed bases (powers_of_gamma_g) appended after them
  size_t stride = 0;   // n_srs + n_extra: entries per window table
  int c = 0, W = 0;
  int T = 0, m = 1;        // window tables kept, bucket sets per MSM (m = ceil(W / T); T = W, m = 1: the full layout)
  size_t max_pairs = 0;    // pairs per bucket pass (0: one pass per MSM)
  // batched-affine levels run before the XYZZ bucket pass (msm_affine.cuh); override: B2M_MSM_AFFINE_LEVELS.
  // Off for a 254-bit Fq: its multiplications are so cheap that the levels' extra memory traffic costs more
  // than the saved multiplications.
  int affine_levels = Fq::N > 8 ? 3 : 0;
  // levels >= 1 (streaming operands): split kernels with the level-wide batch inversion, 32 additions per chain, are faster
  // than the fused kernel at T = 64; level 0 (random gathers) is the other way round.  On H100 the software-pipelined
  // addition pass at 3 CTAs/SM (22) beats the plain one at 4 (21) on these levels; level 0 stays with the plain fused kernel.
  int affine_ctas_upper = 22;  // B2M_MSM_AFFINE_CTAS_UPPER
  int affine_ctas = 4;      // level-kernel variant of level 0 (B2M_MSM_AFFINE_CTAS; the list is at the launch site in msm_impl.cuh)
  size_t affine_min_refs = MSM_AFFINE_MIN_REFS;  // B2M_MSM_AFFINE_MIN_REFS
  int affine_map = 1;       // output -> thread mapping of the levels: 1 = warp-interleaved (coalesced), 0 = blocked; B2M_MSM_AFFINE_MAP
  int affine_T = 64;        // additions per thread (chain) at level 0; B2M_MSM_AFFINE_T sets both
  int affine_T_upper = 32;  // ... at levels >= 1; B2M_MSM_AFFINE_T_UPPER
  int acc_ctas_per_sm = 3;  // resident CTAs of msm_accumulate_kernel per SM (occupancy query)
  DBuf<Affine<Fq>> tables;  // [T][stride]:  tables[j * stride + k] = 2^(c*m*j) * P_(k * world + rank)

  static int pick_window(size_t n);
  // Upload the powers and build the window tables (key-load time).  powers_on_device: `powers` is a device array (the
  // verifier's decoded proof points), copied on the device; single-GPU contexts only.  n_tables (0: all W) and max_pairs
  // (0: no cap) choose a reduced layout; multi-GPU contexts take the full one only.
  Msm(Ctx& cx, const Affine<Fq>* powers, size_t n, const Affine<Fq>* host_extra, size_t n_extra_bases, int window_bits,
      bool powers_on_device = false, int n_tables = 0, size_t max_pairs = 0);

  // sum_i scalars[i] * powers[base_off + i] (+ the `extra` XYZZ terms) -> out_xyzz / out_affine on
  // the device.  `scalars` is a device array, Montgomery form if mont, canonical otherwise.
  void run(const Fr* scalars, bool mont, size_t n, size_t base_off, const XYZZ<Fq>* extra, int n_extra, XYZZ<Fq>* out_xyzz,
           Affine<Fq>* out_affine);
  // Several MSMs at once (the commitments of one prover round): bucket passes back to back, then ONE
  // batched log-depth reduction, so its latency is paid per round instead of per MSM.
  void run_batch(const MsmJob<Fr, Fq>* jobs, int nj);
  // One bucket pass per job (run_batch splits jobs longer than max_pairs into several of these).
  void run_pass(const MsmJob<Fr, Fq>* jobs, int nj);
  // Level-0 ABI bodies (include/b2m.h): host scalars in, host affine point out.
  void run_host(size_t base_off, const uint64_t* scalars, size_t n, uint64_t* out_xy, int* out_is_inf);
  // powers_of_g[i] (affine Montgomery limbs) back to the host: window-0 table entry, from the GPU that holds it
  void read_power(size_t i, uint64_t* out_xy);
  // affine Montgomery points <-> ark-serialize uncompressed bytes (canonical x || y, infinity flag in the last byte)
  static void g1_to_bytes(Ctx& cx, const Affine<Fq>* dev_pts, const uint64_t* host_pts, size_t n, uint8_t* out);
  static void g1_from_bytes(Ctx& cx, const uint8_t* bytes, size_t n, uint64_t* out_xy);
  static void g1_powers_host(Ctx& cx, const uint64_t* g_xy, const uint64_t* beta, size_t n, uint64_t* out);
  // out[i] = scalars[i] * g (canonical host scalars), or beta^(first + i) * g when scalars is null: windowed fixed-base
  // multiplication + batch normalisation [U ark-ec FixedBaseMSM::multi_scalar_mul as KZG10::setup uses it]
  static void fixed_base_host(Ctx& cx, const uint64_t* g_xy, const uint64_t* scalars, const uint64_t* beta, size_t first, size_t n, uint64_t* out);
};

}  // namespace b2m
