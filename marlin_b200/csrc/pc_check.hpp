// Level-1 `PC::check_combinations` for MarlinKZG10 / SonicKZG10, the host bookkeeping [U ark-poly-commit 0.3 marlin_pc /
// sonic_pc check_combinations_individual_opening_challenges -> batch_check]: one set's linear combinations, query set,
// evaluations and opening proofs become per opening point a list of (Fr scalar, G1 base) terms of
//     e(plain + z W, h) * e(-W, beta h) * prod_d e(C_d, beta^-(D-d) h) = 1,
// the equation form of the Marlin verifier (verify_impl.cuh), whose batch check (VerifyItems) folds and bisects the sets.
// Host only: tests/host/pc_check_host_shim.cpp builds it for the CPU tests.
#pragma once
#include <algorithm>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

#include "../../include/b2m.h"
#include "field.cuh"
#include "pairing_host.hpp"  // canonical_lt_modulus

namespace b2m {

// One opening point's equation as terms; bases below the call's shared-base count are shared bases, the rest the item's points
template <class Fr>
struct VerifyTerm {
  Fr c;
  uint32_t base;
};
template <class Fr>
struct VerifyPoint {  // plain + z W against h, W against beta h, bounded[k] against the key's beta^-(D - d_k) h
  std::vector<VerifyTerm<Fr>> plain;
  std::vector<std::pair<size_t, VerifyTerm<Fr>>> bounded;
  Fr z;
  uint32_t w;
};
template <class Fr>
struct VerifyEq {  // one item of a batch check (a Marlin proof, or a Level-1 opening set): one equation per opening point
  std::vector<VerifyPoint<Fr>> pt;
};

// b2m_pc_check_combinations's arguments (include/b2m.h): n sets, flattened; every index inside a set is local to the set
struct PcSets {
  size_t n;
  const size_t* comm_off;  // n + 1
  const uint8_t* comms;
  const int64_t* comm_bounds;
  const int* has_shifted;
  const uint8_t* shifted;
  const size_t* lc_off;       // n + 1
  const size_t* lc_term_off;  // lc_off[n] + 1
  const int64_t* lc_comm;
  const uint64_t* lc_coeff;
  const size_t* point_off;  // n + 1
  const uint64_t* points;
  const uint8_t* w;
  const int* has_random_v;
  const uint8_t* random_v;
  const size_t* query_off;  // n + 1
  const size_t* query_lc;
  const size_t* query_point;
  const uint8_t* evals;
  const uint64_t* challenges;
};

// The PC verifier key's shared bases: g, gamma g, then one MarlinKZG10 shift power powers_of_g[D - d] per enforced bound
enum { PC_S_G, PC_S_GAMMA_G, PC_S_SHIFT };

inline size_t pc_bound_index(const std::vector<uint64_t>& bounds, int64_t d) {
  return (size_t)(std::find(bounds.begin(), bounds.end(), (uint64_t)d) - bounds.begin());
}

// The `Err` cases of upstream check_combinations for set s, decided before any work: "" when there is none.  Offsets must not
// decrease, term, query and point indices must lie in the set, every degree bound must be one the key enforces
// (UnsupportedDegreeBound), a bounded commitment may only be an LC of its own with coefficient one (EquationHasDegreeBounds;
// upstream asserts the coefficient), a query may not repeat (the query set is a set) and every point has a query (one proof per
// queried point).
template <class Fr>
std::string pc_set_error(const PcSets& S, size_t s, const std::vector<uint64_t>& bounds) {
  auto str = [](size_t v) { return std::to_string(v); };
  if (S.comm_off[s + 1] < S.comm_off[s] || S.lc_off[s + 1] < S.lc_off[s] || S.point_off[s + 1] < S.point_off[s] || S.query_off[s + 1] < S.query_off[s])
    return "decreasing offsets";
  const size_t c0 = S.comm_off[s], nc = S.comm_off[s + 1] - c0, l0 = S.lc_off[s], nl = S.lc_off[s + 1] - l0;
  const size_t np = S.point_off[s + 1] - S.point_off[s], q0 = S.query_off[s], nq = S.query_off[s + 1] - q0;
  for (size_t i = 0; i < nc; i++)
    if (S.comm_bounds[c0 + i] >= 0 && pc_bound_index(bounds, S.comm_bounds[c0 + i]) == bounds.size())
      return "commitment " + str(i) + ": degree bound " + std::to_string(S.comm_bounds[c0 + i]) + " is not enforced by the key";
  for (size_t l = 0; l < nl; l++) {
    const size_t t0 = S.lc_term_off[l0 + l], t1 = S.lc_term_off[l0 + l + 1];
    if (t1 < t0) return "decreasing offsets";
    for (size_t t = t0; t < t1; t++) {
      const int64_t c = S.lc_comm[t];
      if (c < -1 || c >= (int64_t)nc) return "LC " + str(l) + " term " + str(t - t0) + " names commitment " + std::to_string(c) + " of " + str(nc);
      if (c < 0 || S.comm_bounds[c0 + c] < 0) continue;
      if (t1 - t0 != 1) return "LC " + str(l) + ": EquationHasDegreeBounds (degree-bounded commitment " + std::to_string(c) + " among " + str(t1 - t0) + " terms)";
      if (memcmp(S.lc_coeff + 4 * t, Fr::one().l, sizeof(Fr)) != 0)
        return "LC " + str(l) + ": the coefficient of degree-bounded commitment " + std::to_string(c) + " is not one";
    }
  }
  std::vector<std::pair<size_t, size_t>> q(nq);
  for (size_t k = 0; k < nq; k++) {
    q[k] = {S.query_point[q0 + k], S.query_lc[q0 + k]};
    if (q[k].second >= nl) return "query " + str(k) + " names LC " + str(q[k].second) + " of " + str(nl);
    if (q[k].first >= np) return "query " + str(k) + " names point " + str(q[k].first) + " of " + str(np);
  }
  std::sort(q.begin(), q.end());
  for (size_t k = 1; k < nq; k++)
    if (q[k] == q[k - 1]) return "query (LC " + str(q[k].second) + ", point " + str(q[k].first) + ") repeats";
  for (size_t j = 0, k = 0; j < np; j++) {
    while (k < nq && q[k].first < j) k++;
    if (k == nq || q[k].first != j) return "point " + str(j) + " has no query";
  }
  return "";
}

// Set s's compressed G1 points in slot order: its commitments, the shifted commitments of MarlinKZG10's bounded commitments
// (where given), then one w per point
inline std::vector<const uint8_t*> pc_set_points(int pc, const PcSets& S, size_t s, size_t fq_bytes) {
  std::vector<const uint8_t*> p;
  for (size_t i = S.comm_off[s]; i < S.comm_off[s + 1]; i++) p.push_back(S.comms + i * fq_bytes);
  if (pc == B2M_PC_MARLIN_KZG10)
    for (size_t i = S.comm_off[s]; i < S.comm_off[s + 1]; i++)
      if (S.comm_bounds[i] >= 0 && S.has_shifted[i]) p.push_back(S.shifted + i * fq_bytes);
  for (size_t j = S.point_off[s]; j < S.point_off[s + 1]; j++) p.push_back(S.w + j * fq_bytes);
  return p;
}

// The equations of set s (which passed pc_set_error): its points are bases base0 + slot (pc_set_points order), the key's shared
// bases PC_S_*.  Per point, LCs in label order take challenge xi^k; a bounded LC under MarlinKZG10 spends a second challenge on
// shifted - v powers_of_g[D - d], under SonicKZG10 it goes against its bound's G2 point; LCTerm::One leaves the evaluation; the
// combined value and random_v go against g and gamma g.  false: malformed (an evaluation or random_v not below r, a bounded
// MarlinKZG10 commitment without its shifted commitment).
template <class Fr>
bool pc_set_equations(int pc, const PcSets& S, size_t s, const std::vector<uint64_t>& bounds, uint32_t base0, VerifyEq<Fr>& E) {
  const bool marlin = pc == B2M_PC_MARLIN_KZG10;
  const size_t c0 = S.comm_off[s], nc = S.comm_off[s + 1] - c0, l0 = S.lc_off[s], nl = S.lc_off[s + 1] - l0;
  const size_t p0 = S.point_off[s], np = S.point_off[s + 1] - p0, q0 = S.query_off[s], nq = S.query_off[s + 1] - q0;
  auto fr_canonical = [](const uint8_t* b, Fr& out) {
    Fr c;
    memcpy(c.l, b, sizeof(c.l));
    if (!canonical_lt_modulus(c)) return false;
    out = Fr::from_canonical(c);
    return true;
  };
  auto fr_mont = [](const uint64_t* p) {
    Fr x;
    memcpy(x.l, p, sizeof(x.l));
    return x;
  };
  std::vector<uint32_t> shifted(nc, 0);
  uint32_t slot = (uint32_t)nc;
  for (size_t i = 0; i < nc && marlin; i++)
    if (S.comm_bounds[c0 + i] >= 0) {
      if (!S.has_shifted[c0 + i]) return false;
      shifted[i] = slot++;
    }
  const uint32_t w0 = slot;
  std::vector<Fr> konst(nl, Fr::zero());      // sum of the LC's LCTerm::One coefficients
  std::vector<int64_t> lc_comm(nl, -1);        // a degree-bounded LC's commitment
  for (size_t l = 0; l < nl; l++)
    for (size_t t = S.lc_term_off[l0 + l]; t < S.lc_term_off[l0 + l + 1]; t++) {
      if (S.lc_comm[t] < 0) konst[l] = konst[l] + fr_mont(S.lc_coeff + 4 * t);
      else if (S.comm_bounds[c0 + S.lc_comm[t]] >= 0) lc_comm[l] = S.lc_comm[t];
    }
  std::vector<std::vector<std::pair<size_t, size_t>>> at(np);  // per point: (LC, query), sorted by LC = label order
  for (size_t k = 0; k < nq; k++) at[S.query_point[q0 + k]].push_back({S.query_lc[q0 + k], k});
  E.pt.assign(np, VerifyPoint<Fr>{});
  const Fr xi = fr_mont(S.challenges + 4 * s);
  for (size_t j = 0; j < np; j++) {
    std::sort(at[j].begin(), at[j].end());
    VerifyPoint<Fr>& pe = E.pt[j];
    Fr ch = Fr::one(), combined = Fr::zero();
    auto next = [&]() {
      const Fr c = ch;
      ch = ch * xi;
      return c;
    };
    for (const auto& lq : at[j]) {
      const size_t l = lq.first;
      Fr v;
      if (!fr_canonical(S.evals + (q0 + lq.second) * sizeof(Fr::l), v)) return false;
      v = v - konst[l];
      const Fr c = next();
      combined = combined + c * v;
      const size_t bidx = lc_comm[l] < 0 ? bounds.size() : pc_bound_index(bounds, S.comm_bounds[c0 + lc_comm[l]]);
      for (size_t t = S.lc_term_off[l0 + l]; t < S.lc_term_off[l0 + l + 1]; t++) {
        if (S.lc_comm[t] < 0) continue;
        const VerifyTerm<Fr> term{c * fr_mont(S.lc_coeff + 4 * t), base0 + (uint32_t)S.lc_comm[t]};
        if (!marlin && lc_comm[l] >= 0) pe.bounded.push_back({bidx, term});
        else pe.plain.push_back(term);
      }
      if (marlin && lc_comm[l] >= 0) {
        const Fr c1 = next();
        pe.plain.push_back(VerifyTerm<Fr>{c1, base0 + shifted[lc_comm[l]]});
        pe.plain.push_back(VerifyTerm<Fr>{(c1 * v).neg(), (uint32_t)(PC_S_SHIFT + bidx)});
      }
    }
    pe.plain.push_back(VerifyTerm<Fr>{combined.neg(), PC_S_G});
    if (S.has_random_v[p0 + j]) {
      Fr rv;
      if (!fr_canonical(S.random_v + (p0 + j) * sizeof(Fr::l), rv)) return false;
      pe.plain.push_back(VerifyTerm<Fr>{rv.neg(), PC_S_GAMMA_G});
    }
    pe.z = fr_mont(S.points + 4 * (p0 + j));
    pe.w = base0 + w0 + (uint32_t)j;
  }
  return true;
}

}  // namespace b2m
