// Radix-2 number-theoretic transform over Fr for sm_90a.
//
// Replaces ark-poly 0.3 `Radix2EvaluationDomain::{fft,ifft}_in_place` [U ark-poly
// src/domain/radix2] behind every `domain.fft / ifft / interpolate /
// evaluate_over_domain` call of the AHP prover [R src/ahp/prover.rs:321-326,350,359,365,
// 427,467,488,532-545,655,681,685].  Same convention: natural-order input and output,
// evals[i] = sum_j c[j] w^(ij) with w = TWO_ADIC_ROOT^(2^(S - log n)); the inverse uses w^-1
// and scales by n^-1.
//
// Structure: decimation-in-frequency, log n stages grouped into passes of up to 8 stages.
// One CTA stages a tile of 2^k strided rows x 8 contiguous columns (256-byte runs, 64 KB)
// in shared memory, runs its k stages there, and writes back; the last pass writes each
// element straight to its bit-reversed slot (32 B = one full sector), so no separate
// permutation pass exists.  Twiddles come from one table w_N^j (j < N/2) for the largest
// domain in use; smaller domains index it with a stride.
#pragma once
#include "common.cuh"
#include "field.cuh"

namespace b2m {

constexpr int NTT_MAX_K = 8;     // stages per pass
constexpr int NTT_THREADS = 256;

template <class Fr>
struct NttTable {
  Fr* tw = nullptr;   // tw[j] = w_N^j, j in [0, N/2)
  int max_log = 0;    // N = 2^max_log
};

template <class Fr>
struct Ntt {
  Ctx* ctx;
  NttTable<Fr> table;
  DBuf<Fr> tw_buf;

  explicit Ntt(Ctx& c);
  static Fr root_of_unity(int log_n);  // w_n = TWO_ADIC_ROOT^(2^(S - log n)), host side
  void ensure_table(int log_n);
  // Transform the 2^log_n elements in `work` (clobbered) into `out` (natural order in and out).
  void run(Fr* work, Fr* out, int log_n, bool inverse);
  // data[i] *= g^i
  void coset_scale(Fr* data, size_t n, const Fr& g);
  // Level-0 ABI body (include/b2m.h b2m_ntt): host buffer in place.
  void run_host(uint64_t* data, unsigned log_n, bool inverse, bool coset);
};

}  // namespace b2m
