// Batched `Marlin::verify` [reference src/lib.rs:315-433] for proofs under one or more index verifier keys of one curve.
// MarlinVerifier holds one key's data; VerifyItems checks a batch of (key, proof) items, b2m_verify_batch being its one-key case.
//
//   1. parse (host)        the `Proof` CanonicalDeserialize framing; evaluations and random_v must be canonical Fr
//   2. decode (GPU)        one thread per compressed G1 point of the whole batch (g1_decode.cuh): flags, x < p, square root,
//                          BLS12-381 subgroup check; the affine points stay in HBM as the MSM bases
//   3. transcript (host)   the verifier's Fiat-Shamir replay, construct_linear_combinations and the check_combinations
//                          bookkeeping of the PC scheme -> per proof and point a list of (Fr scalar, G1 base) terms of
//                              e(plain + z W, h) * e(-W, beta h) * prod_d e(C_d, beta^-(D-d) h) = 1
//   4. batch check         one 128-bit randomiser per (proof, point) from the caller's rng folds every equation into
//                          MSM_A (plain + z W), MSM_B (W) and, for SonicKZG10, one MSM per bound point -- over the checked
//                          proofs' slice of the device-resident bases plus every key's shared bases (index commitments, g,
//                          gamma g, shift powers) with summed scalars -- and one pairing product, checked on the GPU
//                          (pairing_impl.cuh).  Keys with equal (h, beta h) form one G2 group (verify_layout.hpp) with its own
//                          A and B MSMs and its own product; a check passes iff all its products are 1.  The G1 terms under
//                          different keys are independent, so independent randomisers keep the folded check sound.
//   5. bisection           a failing set is split in halves, each checked with fresh randomisers, until every bad proof is
//                          isolated: m bad proofs cost O(m log N) extra checks, made level by level (all checks of a level in
//                          one MSM batch and one pairing launch), so O(log N) rounds
#pragma once
#include <algorithm>
#include <chrono>
#include <cstdint>
#include <cstring>
#include <thread>

#include "capi_types.cuh"
#include "g1_decode.cuh"
#include "pairing_host.hpp"  // g2_prepare: the on-twist check of the key's G2 points
#include "pairing_impl.cuh"
#include "prover_impl.cuh"  // MarlinIndex's ToBytes writers (the transcript encodes commitments as the prover does)
#include "verify.cuh"
#include "verify_layout.hpp"

namespace b2m {

template <class Fq>
__global__ void g1_decode_kernel(const uint8_t* bytes, size_t n, Affine<Fq>* out, int* status) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<Fq> p;
  status[i] = g1_decompress<Fq>(bytes + i * (Fq::N * 4), &p);
  st_words(out + i, p);
}

// The verifier half of a MarlinKZG10 / SonicKZG10 `VerifierKey`, as b2m_vk_create and b2m_pc_vk_create both take it: h and
// beta h must be finite points of the twist; per degree bound, MarlinKZG10's shift power powers_of_g[D - d] (G1 limbs) is
// appended to `shift`, SonicKZG10's beta^-(D - d) h (uncompressed G2) is checked like h.  g2_bytes receives h, beta h and the
// SonicKZG10 points, g2set the same points prepared for the GPU pairing.
template <class Fq>
void pc_key_g2(Ctx& cx, int pc, const uint8_t* h_bytes, const uint8_t* beta_h_bytes, size_t n_bounds, const void* bound_points,
               std::vector<Affine<Fq>>& shift, std::vector<uint8_t>& g2_bytes, std::unique_ptr<PairingG2Set<Fq>>& g2set) {
  constexpr size_t G2_BYTES = 4 * Fq::N * 4;
  G2Prepared<Fq> h, beta_h;
  B2M_REQUIRE(g2_prepare<Fq>(h_bytes, &h) && g2_prepare<Fq>(beta_h_bytes, &beta_h), B2M_ERR_INVALID_ARG,
              "h / beta_h is not a finite point of the G2 curve");
  for (size_t k = 0; k < n_bounds; k++) {
    if (pc == B2M_PC_MARLIN_KZG10) {
      Affine<Fq> p;
      memcpy(&p, static_cast<const uint64_t*>(bound_points) + k * 2 * (Fq::N / 2), sizeof(p));
      shift.push_back(p);
    } else {
      G2Prepared<Fq> q;
      B2M_REQUIRE(g2_prepare<Fq>(static_cast<const uint8_t*>(bound_points) + k * G2_BYTES, &q), B2M_ERR_INVALID_ARG,
                  "neg_powers_of_h[%zu] is not a finite point of the G2 curve", k);
    }
  }
  g2_bytes.assign(h_bytes, h_bytes + G2_BYTES);
  g2_bytes.insert(g2_bytes.end(), beta_h_bytes, beta_h_bytes + G2_BYTES);
  if (pc == B2M_PC_SONIC_KZG10)
    g2_bytes.insert(g2_bytes.end(), static_cast<const uint8_t*>(bound_points), static_cast<const uint8_t*>(bound_points) + n_bounds * G2_BYTES);
  g2set.reset(new PairingG2Set<Fq>(cx, g2_bytes.size() / G2_BYTES, g2_bytes.data()));
}

// Decode n compressed G1 points (FQ_BYTES each, back to back) on the GPU into dst (device); status (host) receives each point's
// g1_decompress status and, when host_pts is given, the decoded points too
template <class Fq>
void decode_g1_bases(Ctx& cx, const std::vector<uint8_t>& bytes, size_t n, Affine<Fq>* dst, std::vector<int>& status, Affine<Fq>* host_pts) {
  status.assign(n, 0);
  if (!n) return;
  DBuf<uint8_t> dbytes(cx, bytes.size());
  DBuf<int> dstatus(cx, n);
  dbytes.upload(bytes.data(), bytes.size());
  g1_decode_kernel<Fq><<<div_up(n, 128), 128, 0, cx.stream>>>(dbytes.p, n, dst, dstatus.p);
  B2M_CHECK_LAUNCH();
  cx.launches++;
  dstatus.download(status.data(), n);
  if (host_pts) B2M_CUDA(cudaMemcpyAsync(host_pts, dst, n * sizeof(Affine<Fq>), cudaMemcpyDeviceToHost, cx.stream));
  cx.sync();
}

// f(i) for i < n on the host's cores: for per-item work that is independent across items
template <class F>
void host_parallel(size_t n, F&& f) {
  const unsigned nt = std::max(1u, std::min(std::thread::hardware_concurrency(), (unsigned)((n + 63) / 64)));
  std::vector<std::thread> pool;
  for (unsigned t = 0; t < nt; t++)
    pool.emplace_back([&, t] {
      for (size_t i = t; i < n; i += nt) f(i);
    });
  for (auto& th : pool) th.join();
}

template <class Fr, class Fq>
struct MarlinVerifier : VerifierBase {
  using Pt = Affine<Fq>;
  using MI = MarlinIndex<Fr, Fq>;
  static constexpr size_t FQ_BYTES = Fq::N * 4, FR_BYTES = Fr::N * 4;
  // the proof's commitments in round order: w, z_a, z_b, mask_poly | t, g_1, h_1 | g_2, h_2
  enum { C_W, C_ZA, C_ZB, C_MASK, C_T, C_G1, C_H1, C_G2, C_H2, N_COMMS };
  // shared bases: the six index commitments (row, col, a_val, b_val, c_val, row_col), g, gamma g, MarlinKZG10 shift powers
  enum { S_ROW, S_COL, S_AVAL, S_BVAL, S_CVAL, S_ROWCOL, S_G, S_GAMMA_G, S_SHIFT };

  Ctx& cx;
  int pc;
  size_t nc, nv, nnz, H, K;
  std::vector<Pt> shared;  // this key's shared bases, at a per-call offset among the MSM's extra bases
  std::vector<uint64_t> bounds;
  size_t bidx_h, bidx_k;  // indices of |H| - 2 and |K| - 2 among the bounds
  std::vector<uint8_t> g2_bytes;            // h, beta_h, then SonicKZG10's beta^-(D - d) h per bound (uncompressed)
  std::unique_ptr<PairingG2Set<Fq>> g2set;  // the same points, prepared for the GPU pairing
  std::vector<uint8_t> vk_bytes;

  static size_t pow2_at_least(size_t n) {
    size_t s = 1;
    while (s < n) s <<= 1;
    return s;
  }
  static Pt pt_from_limbs(const uint64_t* p) {
    Pt r;
    memcpy(&r, p, sizeof(r));
    return r;
  }

  MarlinVerifier(Ctx& c, const VkArgs& a) : cx(c), pc(a.pc), nc(a.num_constraints), nv(a.num_variables), nnz(a.num_non_zero) {
    B2M_REQUIRE(nc == nv, B2M_ERR_NON_SQUARE, "matrices are not square: %zu constraints, %zu variables", nc, nv);
    B2M_REQUIRE(nc >= 2 && nnz >= 2, B2M_ERR_INVALID_ARG, "bad index sizes");
    H = pow2_at_least(nc);
    K = pow2_at_least(nnz);
    for (int i = 0; i < 6; i++) shared.push_back(pt_from_limbs(a.index_comms_xy + i * 2 * (Fq::N / 2)));
    shared.push_back(pt_from_limbs(a.g_xy));
    shared.push_back(pt_from_limbs(a.gamma_g_xy));
    bounds.assign(a.bounds, a.bounds + a.n_bounds);
    bidx_h = bidx_k = a.n_bounds;
    for (size_t k = 0; k < a.n_bounds; k++) {
      if (bounds[k] == H - 2) bidx_h = k;
      if (bounds[k] == K - 2) bidx_k = k;
    }
    B2M_REQUIRE(bidx_h < a.n_bounds && bidx_k < a.n_bounds, B2M_ERR_INVALID_ARG, "the key must carry the degree bounds |H| - 2 = %zu and |K| - 2 = %zu",
                H - 2, K - 2);
    pc_key_g2<Fq>(cx, pc, a.h_bytes, a.beta_h_bytes, a.n_bounds, a.bound_points, shared, g2_bytes, g2set);
    // IndexVerifierKey ToBytes [reference src/data_structures.rs:36-43]: index_info || index_comms
    put_u64(vk_bytes, nv);
    put_u64(vk_bytes, nc);
    put_u64(vk_bytes, nnz);
    for (int i = 0; i < 6; i++) write_commitment(vk_bytes, shared[i], false, Pt::inf());
  }

  size_t g2_points() const { return g2_bytes.size() / (4 * FQ_BYTES); }

  void write_commitment(std::vector<uint8_t>& out, const Pt& comm, bool has_shifted, const Pt& shifted) const {
    MI::put_affine_tobytes(out, comm);
    if (pc == B2M_PC_MARLIN_KZG10) {
      out.push_back(has_shifted ? 1 : 0);
      MI::put_affine_tobytes(out, has_shifted ? shifted : Pt::inf());
    }
  }

  // ---- 1. framing ---------------------------------------------------------------------------------------------
  struct Parsed {
    std::vector<size_t> pt_off;  // byte offset of every compressed point, in slot order
    int comm[N_COMMS], shifted[N_COMMS], w[2];  // slots (shifted: -1 when absent)
    Fr evals[4];                 // g_1(beta), g_2(gamma), t(beta), z_b(beta)
    bool has_rv[2];
    Fr rv[2];
  };
  bool parse(const uint8_t* d, size_t len, Parsed& P) const {
    size_t off = 0;
    auto need = [&](size_t n) { return off + n <= len; };
    auto u64 = [&](uint64_t& v) {
      if (!need(8)) return false;
      v = 0;
      for (int i = 0; i < 8; i++) v |= (uint64_t)d[off + i] << (8 * i);
      off += 8;
      return true;
    };
    auto byte = [&](uint8_t& v) {
      if (!need(1)) return false;
      v = d[off++];
      return true;
    };
    auto point = [&]() {
      if (!need(FQ_BYTES)) return -1;
      P.pt_off.push_back(off);
      off += FQ_BYTES;
      return (int)P.pt_off.size() - 1;
    };
    auto fr = [&](Fr& out) {
      if (!need(FR_BYTES)) return false;
      Fr c;
      memcpy(c.l, d + off, FR_BYTES);
      off += FR_BYTES;
      if (!canonical_lt_modulus(c)) return false;
      out = Fr::from_canonical(c);
      return true;
    };
    uint64_t v;
    uint8_t b;
    const uint64_t round_sizes[3] = {4, 3, 2};
    if (!u64(v) || v != 3) return false;
    int k = 0;
    for (int r = 0; r < 3; r++) {
      if (!u64(v) || v != round_sizes[r]) return false;
      for (uint64_t i = 0; i < round_sizes[r]; i++, k++) {
        if ((P.comm[k] = point()) < 0) return false;
        P.shifted[k] = -1;
        if (pc == B2M_PC_MARLIN_KZG10) {
          if (!byte(b) || b > 1) return false;
          if (b && (P.shifted[k] = point()) < 0) return false;
        }
      }
    }
    if (!u64(v) || v != 4) return false;
    for (int i = 0; i < 4; i++)
      if (!fr(P.evals[i])) return false;
    if (!u64(v) || v != 3) return false;  // three ProverMsg::EmptyMessage
    for (int i = 0; i < 3; i++)
      if (!byte(b) || b != 0) return false;
    if (!u64(v) || v != 2) return false;
    for (int j = 0; j < 2; j++) {
      if ((P.w[j] = point()) < 0) return false;
      if (!byte(b) || b > 1) return false;
      P.has_rv[j] = b == 1;
      if (b && !fr(P.rv[j])) return false;
    }
    if (!byte(b) || b != 0) return false;  // BatchLCProof.evals = None
    return off == len;
  }

  // ---- 3. the verifier's transcript and check_combinations bookkeeping ---------------------------------------------
  using Term = VerifyTerm<Fr>;
  using PointEq = VerifyPoint<Fr>;
  using ProofEq = VerifyEq<Fr>;  // two points: beta and gamma

  Fr sample_outside_h(FiatShamir& fs) const {
    for (;;) {
      Fr t = field_rand<Fr>(fs);
      if (t.pow_u64(H) != Fr::one()) return t;
    }
  }
  static Fr fr_u128(uint64_t lo, uint64_t hi) {
    Fr c = Fr::zero();
    c.l[0] = (uint32_t)lo; c.l[1] = (uint32_t)(lo >> 32); c.l[2] = (uint32_t)hi; c.l[3] = (uint32_t)(hi >> 32);
    return Fr::from_canonical(c);
  }

  // false: the proof is rejected without a pairing (a degree-bounded commitment without its shifted half).  The proof's points
  // are bases base0 + slot, this key's shared bases sbase0 + S_*.
  bool equations(const Parsed& P, const Pt* pts, uint32_t base0, uint32_t sbase0, const uint64_t* input, size_t n_input, ProofEq& E) const {
    const bool marlin = pc == B2M_PC_MARLIN_KZG10;
    if (marlin && (P.shifted[C_G1] < 0 || P.shifted[C_G2] < 0)) return false;
    const Fr one = Fr::one();
    // public input padded to |X| - 1 [reference lib.rs:323-333], X = the domain of the formatted input
    const size_t X = pow2_at_least(n_input + 1);
    std::vector<Fr> formatted(X, Fr::zero());
    formatted[0] = one;
    for (size_t i = 0; i < n_input; i++) memcpy(formatted[i + 1].l, input + 4 * i, sizeof(Fr));
    std::vector<uint8_t> init;
    const char* proto = "MARLIN-2019";
    init.insert(init.end(), proto, proto + 11);
    init.insert(init.end(), vk_bytes.begin(), vk_bytes.end());
    for (size_t i = 1; i < X; i++) MI::put_fr_canonical(init, formatted[i]);
    FiatShamir fs(init);
    auto absorb_round = [&](int first, int count) {
      std::vector<uint8_t> bytes;
      for (int k = first; k < first + count; k++)
        write_commitment(bytes, pts[P.comm[k]], P.shifted[k] >= 0, P.shifted[k] >= 0 ? pts[P.shifted[k]] : Pt::inf());
      fs.absorb(bytes);
    };
    absorb_round(0, 4);
    const Fr alpha = sample_outside_h(fs);
    const Fr eta_a = field_rand<Fr>(fs), eta_b = field_rand<Fr>(fs), eta_c = field_rand<Fr>(fs);
    absorb_round(4, 3);
    const Fr beta = sample_outside_h(fs);
    absorb_round(7, 2);
    const Fr gamma = field_rand<Fr>(fs);
    {
      std::vector<uint8_t> eb;
      for (const Fr& e : P.evals) MI::put_fr_canonical(eb, e);
      fs.absorb(eb);
    }
    uint64_t lo = fs.next_u64(), hi = fs.next_u64();
    const Fr xi = fr_u128(lo, hi);
    const Fr g1_b = P.evals[0], g2_g = P.evals[1], t_b = P.evals[2], zb_b = P.evals[3];

    // construct_linear_combinations [reference src/ahp/mod.rs:110-221]
    const Fr v_h_alpha = alpha.pow_u64(H) - one, v_h_beta = beta.pow_u64(H) - one;
    Fr r_alpha_at_beta = (v_h_alpha - v_h_beta) * (alpha - beta).inverse_fast();
    if (alpha == beta) r_alpha_at_beta = Fr::from_u64(H) * alpha.pow_u64(H - 1);
    const Fr v_x_beta = beta.pow_u64(X) - one;
    // x(beta) = sum_i L_i(beta) x_i with L_i(beta) = v_X(beta) w^i / (|X| (beta - w^i)); beta is outside H, which holds X
    Fr omega;
    for (int i = 0; i < Fr::N; i++) omega.l[i] = Fr::Params::root(i);
    for (size_t s = X; s < ((size_t)1 << Fr::Params::TWO_ADICITY); s <<= 1) omega = omega.sqr();
    Fr x_at_beta = Fr::zero(), wi = one;
    for (size_t i = 0; i < X; i++) {
      if (!formatted[i].is_zero()) x_at_beta = x_at_beta + formatted[i] * wi * (beta - wi).inverse_fast();
      wi = wi * omega;
    }
    x_at_beta = x_at_beta * v_x_beta * Fr::from_u64(X).inverse_fast();
    const Fr c_za = r_alpha_at_beta * (eta_a + eta_c * zb_b);
    const Fr c_w = (t_b * v_x_beta).neg(), c_h1 = v_h_beta.neg();
    // LCTerm::One constants leave the LC's value: outer_sumcheck evaluates to 0, so its value is minus the constants
    const Fr v_outer = t_b * x_at_beta + beta * g1_b - r_alpha_at_beta * eta_b * zb_b;
    const Fr vv = v_h_alpha * v_h_beta;
    const Fr v_k_gamma = gamma.pow_u64(K) - one;
    const Fr bscale = gamma * g2_g + t_b * Fr::from_u64(K).inverse_fast();
    const Fr v_inner = bscale * alpha * beta;

    // check_combinations [U ark-poly-commit marlin_pc / sonic_pc]: per point, labels in BTreeSet order,
    // challenge xi^k, MarlinKZG10 spending a second challenge on each degree-bounded LC
    auto base = [&](int slot) { return base0 + (uint32_t)slot; };
    E.pt.resize(2);
    for (int j = 0; j < 2; j++) {
      PointEq& pe = E.pt[j];
      Fr ch = one, combined = Fr::zero();
      auto next = [&]() { Fr c = ch; ch = ch * xi; return c; };
      auto bounded_lc = [&](int comm, Fr v, size_t bidx) {  // the single polynomial g_1 / g_2
        const Fr c0 = next();
        combined = combined + c0 * v;
        if (!marlin) {
          pe.bounded.push_back({bidx, Term{c0, base(P.comm[comm])}});
          return;
        }
        pe.plain.push_back(Term{c0, base(P.comm[comm])});
        const Fr c1 = next();  // c1 (shifted - v powers_of_g[D - d])
        pe.plain.push_back(Term{c1, base(P.shifted[comm])});
        pe.plain.push_back(Term{(c1 * v).neg(), sbase0 + (uint32_t)(S_SHIFT + bidx)});
      };
      auto plain_lc = [&](std::initializer_list<std::pair<Fr, uint32_t>> terms, Fr v) {
        const Fr c = next();
        combined = combined + c * v;
        for (const auto& t : terms) pe.plain.push_back(Term{c * t.first, t.second});
      };
      if (j == 0) {  // beta: g_1, outer_sumcheck, t, z_b
        pe.z = beta;
        bounded_lc(C_G1, g1_b, bidx_h);
        plain_lc({{one, base(P.comm[C_MASK])}, {c_za, base(P.comm[C_ZA])}, {c_w, base(P.comm[C_W])}, {c_h1, base(P.comm[C_H1])}}, v_outer);
        plain_lc({{one, base(P.comm[C_T])}}, t_b);
        plain_lc({{one, base(P.comm[C_ZB])}}, zb_b);
      } else {  // gamma: g_2, inner_sumcheck
        pe.z = gamma;
        bounded_lc(C_G2, g2_g, bidx_k);
        plain_lc({{eta_a * vv, sbase0 + S_AVAL}, {eta_b * vv, sbase0 + S_BVAL}, {eta_c * vv, sbase0 + S_CVAL}, {bscale * alpha, sbase0 + S_ROW},
                  {bscale * beta, sbase0 + S_COL}, {bscale.neg(), sbase0 + S_ROWCOL}, {v_k_gamma.neg(), base(P.comm[C_H2])}},
                 v_inner);
      }
      pe.plain.push_back(Term{combined.neg(), sbase0 + S_G});
      if (P.has_rv[j]) pe.plain.push_back(Term{P.rv[j].neg(), sbase0 + S_GAMMA_G});
      pe.w = base(P.w[j]);
    }
    return true;
  }

  void verify_multi(size_t n_keys, VerifierBase* const* keys, size_t n, const uint32_t* key_of, const uint64_t* const* inputs,
                    const size_t* n_inputs, const uint8_t* const* proofs, const size_t* lens, b2m_rng* rng, int* verdicts) override;
};

// ---- 4. + 5. randomised checks, the bisection tree level by level ---------------------------------------------------------
template <class Fr, class Fq>
struct VerifyItems {
  using V = MarlinVerifier<Fr, Fq>;
  using Pt = Affine<Fq>;
  using Clock = std::chrono::steady_clock;
  static double ms_since(Clock::time_point t) { return std::chrono::duration<double, std::milli>(Clock::now() - t).count(); }

  Ctx& cx;
  std::vector<const V*> keys;  // the call's distinct keys
  std::vector<uint32_t> sbase;  // per key: its first shared base
  std::vector<Pt> shared;       // every key's shared bases, concatenated
  std::unique_ptr<Msm<Fr, Fq>> msm;  // bases: the proofs' points; extra bases: the shared ones
  std::vector<typename V::ProofEq> eqs;
  std::vector<uint32_t> key;         // per equation: its key
  std::vector<size_t> pt_lo, pt_hi;  // per equation: its proof's points [lo, hi) among the proof points
  double ms_fold = 0, ms_msm = 0, ms_pairing = 0, ms_first = 0;
  int checks = 0, products = 0;

  explicit VerifyItems(Ctx& c) : cx(c) {}

  // A node is a range [a, b) of equations (contiguous in item order, so its proofs' points are one slice of the bases).  The
  // root is checked; a failing node of one proof is a bad proof, a failing larger node has both halves checked.  That is the
  // depth-first bisection's set of checks, with the same randomisers per check (two 128-bit ones per proof), so the rng ends at
  // the same position; they are only drawn level by level.  A check has one pairing product per G2 group among its proofs:
  // [A_g against h_g, -B_g against beta h_g, then group g's SonicKZG10 slots], and passes iff all of them are 1.  All checks
  // of a level run their MSMs as one Msm::run_batch sequence (each MSM over its node's slice plus the shared bases) and their
  // products as one PairingG2Set::check launch.
  void resolve(const G2Layout& L, PairingG2Set<Fq>& g2, const std::vector<size_t>& proof_of, ZkSource<b2m_rng>& rng, int* verdicts) {
    const size_t S = shared.size();
    std::vector<std::pair<size_t, size_t>> level{{0, eqs.size()}};
    std::vector<size_t> prod_of_group(L.n_groups), job_of_point(L.src.size());
    bool first = true;
    while (!level.empty()) {
      const Clock::time_point t_level = Clock::now();
      // scalars: per MSM, its node's slice (len values) then the S shared bases
      std::vector<Fr> sc;
      std::vector<size_t> job_off, job_len, job_lo;
      struct Pair {
        size_t job;
        uint32_t g2;
        bool neg;  // -W against beta h
      };
      std::vector<std::vector<Pair>> prods;  // the level's products
      std::vector<size_t> node_prod{0};      // node nd's products: [node_prod[nd], node_prod[nd + 1])
      for (size_t nd = 0; nd < level.size(); nd++) {
        const size_t a = level[nd].first, b = level[nd].second, lo = pt_lo[a], len = pt_hi[b - 1] - lo;
        auto new_job = [&]() {
          job_off.push_back(sc.size());
          job_len.push_back(len);
          job_lo.push_back(lo);
          sc.resize(sc.size() + len + S, Fr::zero());
          return job_off.size() - 1;
        };
        auto at = [&](size_t job, uint32_t base) -> Fr& { return base < S ? sc[job_off[job] + len + base] : sc[job_off[job] + (base - S - lo)]; };
        std::fill(prod_of_group.begin(), prod_of_group.end(), SIZE_MAX);
        std::fill(job_of_point.begin(), job_of_point.end(), SIZE_MAX);
        for (size_t i = a; i < b; i++) {
          const std::vector<uint32_t>& kp = L.point[key[i]];
          size_t& pg = prod_of_group[L.group[key[i]]];
          if (pg == SIZE_MAX) {  // plain + z W against h, W against beta h
            pg = prods.size();
            const size_t ja = new_job(), jb = new_job();
            prods.push_back({Pair{ja, kp[0], false}, Pair{jb, kp[1], true}});
          }
          const size_t ja = prods[pg][0].job, jb = prods[pg][1].job;
          for (const auto& pe : eqs[i].pt) {
            uint64_t rlo = rng.next_u64(), rhi = rng.next_u64();
            const Fr r = V::fr_u128(rlo, rhi);
            for (const auto& t : pe.plain) at(ja, t.base) = at(ja, t.base) + r * t.c;
            at(ja, pe.w) = at(ja, pe.w) + r * pe.z;
            at(jb, pe.w) = at(jb, pe.w) + r;
            for (const auto& bt : pe.bounded) {
              const uint32_t q = kp[2 + bt.first];
              if (job_of_point[q] == SIZE_MAX) {
                job_of_point[q] = new_job();
                prods[pg].push_back(Pair{job_of_point[q], q, false});
              }
              at(job_of_point[q], bt.second.base) = at(job_of_point[q], bt.second.base) + r * bt.second.c;
            }
          }
        }
        node_prod.push_back(prods.size());
      }
      ms_fold += ms_since(t_level);
      Clock::time_point t0 = Clock::now();
      for (Fr& x : sc) x = x.to_canonical();
      const size_t nj = job_off.size();
      DBuf<Fr> dsc(cx, sc.size());
      DBuf<Pt> dres(cx, nj);
      dsc.upload(sc.data(), sc.size());
      for (size_t j0 = 0; j0 < nj; j0 += MSM_MAX_BATCH) {
        MsmJob<Fr, Fq> jobs[MSM_MAX_BATCH];
        const int m = (int)std::min<size_t>(MSM_MAX_BATCH, nj - j0);
        for (int k = 0; k < m; k++) {
          const size_t j = j0 + k;
          jobs[k] = MsmJob<Fr, Fq>{dsc.p + job_off[j], false, job_len[j], job_lo[j], dsc.p + job_off[j] + job_len[j], S, 0, nullptr, 0, nullptr,
                                   dres.p + j};
        }
        msm->run_batch(jobs, m);
      }
      std::vector<Pt> res(nj);
      dres.download(res.data(), nj);
      ms_msm += ms_since(t0);
      t0 = Clock::now();
      std::vector<Pt> g1;
      std::vector<uint32_t> g2i;
      std::vector<size_t> off{0};
      for (const auto& pr : prods) {
        for (const Pair& p : pr) {
          const Pt& q = res[p.job];
          g1.push_back(p.neg ? Pt{q.x, q.y.neg()} : q);  // (infinity stays (0, 0))
          g2i.push_back(p.g2);
        }
        off.push_back(g1.size());
      }
      std::vector<int> ok(prods.size());
      g2.check(prods.size(), off.data(), reinterpret_cast<const uint64_t*>(g1.data()), g2i.data(), ok.data());
      ms_pairing += ms_since(t0);
      checks += (int)level.size();
      products += (int)prods.size();
      std::vector<std::pair<size_t, size_t>> next;
      for (size_t nd = 0; nd < level.size(); nd++) {
        const size_t a = level[nd].first, b = level[nd].second;
        if (std::all_of(ok.begin() + node_prod[nd], ok.begin() + node_prod[nd + 1], [](int v) { return v == 1; })) {
          for (size_t i = a; i < b; i++) verdicts[proof_of[i]] = 1;
        } else if (b - a == 1) {
          verdicts[proof_of[a]] = 0;
        } else {
          const size_t half = (b - a) / 2;
          next.push_back({a, a + half});
          next.push_back({a + half, b});
        }
      }
      if (first) ms_first = ms_since(t_level);
      first = false;
      level.swap(next);
    }
  }

  // proof i under call key key_of[i] of n_keys
  void run(size_t n_keys, VerifierBase* const* vks, size_t n, const uint32_t* key_of, const uint64_t* const* inputs, const size_t* n_inputs,
           const uint8_t* const* proofs, const size_t* lens, b2m_rng* rng, int* verdicts) {
    constexpr size_t FQ_BYTES = V::FQ_BYTES;
    Clock::time_point t_all = Clock::now(), t0 = t_all;
    ZkSource<b2m_rng> zr(rng);
    // the distinct keys and their shared bases
    std::vector<uint32_t> uniq(n_keys);
    for (size_t k = 0; k < n_keys; k++) {
      const V* v = static_cast<const V*>(vks[k]);
      uniq[k] = (uint32_t)(std::find(keys.begin(), keys.end(), v) - keys.begin());
      if (uniq[k] < keys.size()) continue;
      keys.push_back(v);
      sbase.push_back((uint32_t)shared.size());
      shared.insert(shared.end(), v->shared.begin(), v->shared.end());
    }
    const size_t S = shared.size();
    // 1. framing
    std::vector<typename V::Parsed> parsed(n);
    std::vector<uint32_t> first(n, 0);
    std::vector<uint8_t> bytes;
    size_t n_pts = 0;
    for (size_t i = 0; i < n; i++) {
      verdicts[i] = -1;
      if (!proofs[i] || !keys[uniq[key_of[i]]]->parse(proofs[i], lens[i], parsed[i])) continue;
      verdicts[i] = 0;
      first[i] = (uint32_t)(S + n_pts);
      for (size_t off : parsed[i].pt_off) bytes.insert(bytes.end(), proofs[i] + off, proofs[i] + off + FQ_BYTES);
      n_pts += parsed[i].pt_off.size();
    }
    // 2. decode on the GPU, straight into the MSM base array behind the shared bases
    DBuf<Pt> bases(cx, S + n_pts);
    std::vector<Pt> host_pts(n_pts);
    std::vector<int> status;
    bases.upload(shared.data(), S);
    decode_g1_bases<Fq>(cx, bytes, n_pts, bases.p + S, status, host_pts.data());
    const double ms_decode = ms_since(t0);
    // 3. transcript and equations
    t0 = Clock::now();
    std::vector<typename V::ProofEq> all_eqs(n);
    std::vector<char> has_eq(n, 0);
    for (size_t i = 0; i < n; i++) {
      if (verdicts[i] < 0) continue;
      const size_t p0 = first[i] - S;
      for (size_t k = 0; k < parsed[i].pt_off.size(); k++)
        if (status[p0 + k] != G1_OK) verdicts[i] = -1;
    }
    host_parallel(n, [&](size_t i) {  // O(1) Fr work + O(|X|) per proof
      if (verdicts[i] != 0) return;
      const uint32_t u = uniq[key_of[i]];
      has_eq[i] = keys[u]->equations(parsed[i], host_pts.data() + (first[i] - S), first[i], sbase[u], inputs[i], n_inputs[i], all_eqs[i]);
    });
    std::vector<size_t> proof_of;
    for (size_t i = 0; i < n; i++) {
      if (!has_eq[i]) continue;  // verdict -1 (malformed) or 0 (no shifted commitment for a bounded polynomial)
      proof_of.push_back(i);
      eqs.push_back(std::move(all_eqs[i]));
      key.push_back(uniq[key_of[i]]);
      pt_lo.push_back(first[i] - S);
      pt_hi.push_back(first[i] - S + parsed[i].pt_off.size());
    }
    const double ms_transcript = ms_since(t0);
    // 4. + 5., with the call's G2 set: every group's points, copied from the keys' prepared lines
    std::vector<std::pair<const uint8_t*, size_t>> kg2;
    for (const V* v : keys) kg2.push_back({v->g2_bytes.data(), v->g2_points()});
    const G2Layout L = g2_layout(kg2, 4 * FQ_BYTES);
    double ms_g2 = 0, ms_tables = 0, ms_checks = 0;
    if (!eqs.empty()) {
      t0 = Clock::now();
      std::vector<std::pair<const PairingG2Set<Fq>*, size_t>> src;
      for (const auto& s : L.src) src.push_back({keys[s.first]->g2set.get(), s.second});
      PairingG2Set<Fq> g2(cx, src);
      ms_g2 = ms_since(t0);
      t0 = Clock::now();
      msm.reset(new Msm<Fr, Fq>(cx, bases.p + S, n_pts, shared.data(), S, 0, true));
      ms_tables = ms_since(t0);
      t0 = Clock::now();
      resolve(L, g2, proof_of, zr, verdicts);
      ms_checks = ms_since(t0);
    }
    zr.commit_position();
    // msm_ms / pairing_ms cover every check; bisection_ms is the time of the checks after the first
    const std::string json = fmt(
        "{\"proofs\": %zu, \"points\": %zu, \"decode_ms\": %.4f, \"transcript_ms\": %.4f, \"g2_set_ms\": %.4f, \"msm_tables_ms\": %.4f, "
        "\"msm_ms\": %.4f, \"pairing_ms\": %.4f, \"first_check_ms\": %.4f, \"bisection_ms\": %.4f, \"checks\": %d, \"keys\": %zu, "
        "\"g2_groups\": %zu, \"products\": %d, \"total_ms\": %.4f}",
        n, n_pts, ms_decode, ms_transcript, ms_g2, ms_tables, ms_msm, ms_pairing, ms_first, ms_checks - ms_first, checks, keys.size(), L.n_groups,
        products, ms_since(t_all));
    for (size_t k = 0; k < n_keys; k++) vks[k]->timings_json = json;
  }
};

template <class Fr, class Fq>
void MarlinVerifier<Fr, Fq>::verify_multi(size_t n_keys, VerifierBase* const* keys, size_t n, const uint32_t* key_of, const uint64_t* const* inputs,
                                          const size_t* n_inputs, const uint8_t* const* proofs, const size_t* lens, b2m_rng* rng, int* verdicts) {
  VerifyItems<Fr, Fq>(cx).run(n_keys, keys, n, key_of, inputs, n_inputs, proofs, lens, rng, verdicts);
}

}  // namespace b2m
