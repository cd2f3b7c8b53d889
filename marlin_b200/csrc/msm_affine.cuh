// Batched-affine bucket levels for the MSM (csrc/msm_impl.cuh run_batch).
//
// The references of one MSM are sorted by bucket.  Level l holds cnt_l[b] affine points of bucket b at
// positions [off_l[b], off_l[b + 1]); level 0 is the sorted reference list itself (points = +-table entries).
// One level adds the points of every bucket in pairs: cnt_(l+1)[b] = ceil(cnt_l[b] / 2), output j of bucket b
// = point 2j + point 2j + 1 (or a copy of point 2j when the count is odd).  All additions of a level are
// independent, so they are done in AFFINE coordinates with the slopes' denominators inverted together
// (Montgomery's trick): 6 field multiplications per addition instead of 10 for an XYZZ mixed addition.
// A light plan pass resolves which two points make each output.  A thread then owns T outputs (warp-interleaved: the 32
// lanes of a warp own 32 T consecutive outputs, so every step of a warp touches 32 adjacent outputs): pass 1 multiplies
// the denominators up (prefix products to a scratch array), the chain product is inverted, pass 2 walks back and writes
// the sums.  After a few levels the remaining points (n / 2^levels) go through the XYZZ bucket pass, which balances any
// bucket-size distribution.
//
// Forms of the arithmetic kernel, all byte-identical in their results (selectable at run time, msm_impl.cuh launch site):
//   * fused (aff_level_thread): both passes and one binary-Euclid inversion (field.cuh inverse_fast) per thread -- the
//     default for level 0, whose operands are random gathers from the window tables;
//   * branch-free and software-pipelined (aff_level_thread_sp, PHASE 0);
//   * split into two kernels (PHASE 1 + 2, or PHASE 3 + 2 with ONE batch inversion of all chain products of the level in
//     between: msm_impl.cuh fq_batch_inverse_kernel) -- the default for the streaming levels >= 1.
//
// Host/device shared: tests/host builds this with g++ (carry flag emulated) and checks it against the oracle.
#pragma once
#include "curve.cuh"
#ifdef __CUDACC__
#include "devmem.cuh"
#else
struct uint2 {
  uint32_t x, y;
};
struct uint4 {
  uint32_t x, y, z, w;
};
#endif

namespace b2m {

constexpr uint32_t AFF_BKT_BITS = 24;  // == MSM_BKT_BITS (msm.cuh): reference = {table index | sign << 31, bucket | window << 24}

template <class Fq>
struct AffLevel {
  // level-0 source: position i is the point +-tables[window * table_stride + index] named by sorted[i]
  const Affine<Fq>* tables;
  size_t table_stride;
  const uint2* sorted;
  // level >= 1 source: position i is in[i]
  const Affine<Fq>* in;
  const uint32_t* off_in;   // [B + 1] bucket starts of the input level (off_in[B] = number of points)
  const uint32_t* off_out;  // [B + 1] bucket starts of the output level
  uint32_t B;
  Affine<Fq>* out;
  uint2* out_refs;  // last level only (else null): {position, bucket} references for the XYZZ pass over `out`
  Fq* pref;         // [T][nthreads] running denominator products
  uint4* meta;      // [T][nthreads] the plan: {P index | negate << 31, Q index | negate << 31, bucket, has Q}
  uint32_t T, nthreads;
  // Output -> thread mapping.  lane_step == 1 ("blocked"): thread t owns the T consecutive outputs [t T, t T + T).
  // lane_step == 32 ("interleaved", nthreads a multiple of 32): the 32 threads of a warp own 32 T consecutive outputs,
  // lane l taking l, l + 32, l + 64, ... -- at every step the lanes of a warp then touch 32 ADJACENT outputs, so the
  // level's output stores and (levels >= 1) its operand loads are whole contiguous runs (3 KB / 6 KB per warp and step)
  // instead of 32 streams 6 KB apart, which DRAM sees as random 32-byte accesses.
  uint32_t lane_step;
  Fq* inv;  // [nthreads] chain inverses (split form: written by the phase-1 kernel, read by the phase-2 kernel)
};

struct AffMap {
  uint32_t o0, step, cnt;  // outputs o0 + k * step, k < cnt
};
template <class Fq>
B2M_HD AffMap aff_map(const AffLevel<Fq>& A, uint32_t t, uint32_t total) {
  AffMap m;
  m.step = A.lane_step;
  uint64_t o0;
  if (A.lane_step == 1) {
    o0 = (uint64_t)t * A.T;
  } else {
    o0 = (uint64_t)(t / A.lane_step) * A.lane_step * A.T + (t % A.lane_step);
  }
  if (o0 >= total) {
    m.o0 = 0;
    m.cnt = 0;
    return m;
  }
  m.o0 = (uint32_t)o0;
  const uint32_t left = (total - m.o0 + m.step - 1) / m.step;
  m.cnt = left < A.T ? left : A.T;
  return m;
}

#if defined(__CUDA_ARCH__)
#define B2M_AFF_LDG(p) ldg_words(p)
#define B2M_AFF_LD(p) ld_words(p)
#define B2M_AFF_ST(p, v) st_words(p, v)
#define B2M_AFF_LDG32(p) __ldg(p)
#else
#define B2M_AFF_LDG(p) (*(p))
#define B2M_AFF_LD(p) (*(p))
#define B2M_AFF_ST(p, v) (*(p) = (v))
#define B2M_AFF_LDG32(p) (*(p))
#endif

// first index in off[0 .. n] whose value is > v, minus one: the (non-empty) bucket holding position v
B2M_HD uint32_t aff_bucket_of(const uint32_t* off, uint32_t n, uint32_t v) {
  uint32_t lo = 0, hi = n;  // invariant: off[lo] <= v < off[hi]  (off[0] = 0, off[n] = total > v)
  while (hi - lo > 1) {
    uint32_t mid = (lo + hi) >> 1;
    if (B2M_AFF_LDG32(off + mid) <= v) lo = mid; else hi = mid;
  }
  return lo;
}

// ---- plan: which two input points make output o (a light, latency-bound pass kept out of the arithmetic kernel) ----
// Thread t plans the outputs [t * T, t * T + T): meta[k][t] = {index of P, index of Q, bucket, has Q}; the indices
// address `tables` (level 0, resolved from the sorted references, with the sign in bit 31) or `in` (later levels).
template <class Fq, bool L0>
B2M_HD void aff_plan_thread(const AffLevel<Fq>& A, uint32_t t) {
  const uint32_t total = B2M_AFF_LDG32(A.off_out + A.B);
  const AffMap mp = aff_map(A, t, total);
  if (!mp.cnt) return;
  uint32_t b = aff_bucket_of(A.off_out, A.B, mp.o0);
  uint32_t b_start = B2M_AFF_LDG32(A.off_out + b), b_end = B2M_AFF_LDG32(A.off_out + b + 1);
  for (uint32_t k = 0; k < mp.cnt; k++) {
    const uint32_t o = mp.o0 + k * mp.step;
    if (o >= b_end) {
      // next bucket holding `o`: a short walk (the common case: a few buckets ahead), else search -- a stride of 32
      // outputs, or a run of empty buckets, can skip arbitrarily far
      int steps = 0;
      do {
        b++;
        b_end = B2M_AFF_LDG32(A.off_out + b + 1);
      } while (o >= b_end && ++steps < 8);
      if (o >= b_end) {
        b = aff_bucket_of(A.off_out, A.B, o);
        b_end = B2M_AFF_LDG32(A.off_out + b + 1);
      }
      b_start = B2M_AFF_LDG32(A.off_out + b);
    }
    const uint32_t in_start = B2M_AFF_LDG32(A.off_in + b), in_end = B2M_AFF_LDG32(A.off_in + b + 1);
    const uint32_t i0 = in_start + 2u * (o - b_start);
    const bool pair = i0 + 1u < in_end;
    uint4 m;
    if (L0) {
      const uint2 r0 = B2M_AFF_LDG32(A.sorted + i0);
      m.x = (uint32_t)((size_t)(r0.y >> AFF_BKT_BITS) * A.table_stride + (r0.x & 0x7fffffffu)) | (r0.x & 0x80000000u);
      m.y = m.x;
      if (pair) {
        const uint2 r1 = B2M_AFF_LDG32(A.sorted + i0 + 1u);
        m.y = (uint32_t)((size_t)(r1.y >> AFF_BKT_BITS) * A.table_stride + (r1.x & 0x7fffffffu)) | (r1.x & 0x80000000u);
      }
    } else {
      m.x = i0;
      m.y = pair ? i0 + 1u : i0;
    }
    m.z = b;
    m.w = pair ? 1u : 0u;
    A.meta[(size_t)k * A.nthreads + t] = m;
  }
}

template <class Fq>
B2M_HD Fq aff_ldx(const Affine<Fq>* base, uint32_t ref) {
  return B2M_AFF_LDG(&base[ref & 0x7fffffffu].x);
}
template <class Fq>
B2M_HD Affine<Fq> aff_ld(const Affine<Fq>* base, uint32_t ref) {
  const Affine<Fq>* p = base + (ref & 0x7fffffffu);
  Affine<Fq> r;
  r.x = B2M_AFF_LDG(&p->x);
  r.y = B2M_AFF_LDG(&p->y);
  return r;
}
template <class Fq>
B2M_HD Affine<Fq> aff_signed(Affine<Fq> p, uint32_t ref) {
  if (ref >> 31) p.y = p.y.neg();
  return p;
}

enum AffKind : uint32_t { AFF_COPY_P = 0, AFF_COPY_Q = 1, AFF_INF = 2, AFF_ADD = 3, AFF_DBL = 4 };

// P + Q: which formula, and the denominator of its slope (AFF_ADD / AFF_DBL only).
template <class Fq>
B2M_HD AffKind aff_classify(const Affine<Fq>& P, const Affine<Fq>& Q, Fq* den) {
  if (P.is_inf()) return AFF_COPY_Q;
  if (Q.is_inf()) return AFF_COPY_P;
  if (P.x == Q.x) {
    if (P.y == Q.y && !P.y.is_zero()) {
      *den = P.y.dbl();
      return AFF_DBL;
    }
    return AFF_INF;  // Q = -P (or a 2-torsion point doubled)
  }
  *den = Q.x - P.x;
  return AFF_ADD;
}

// ---- arithmetic: thread t adds the planned pairs of its T outputs with one shared inversion -----------------------
// PF: load the next iteration's operands before the current iteration's multiplications (costs ~50 registers, so fewer
// resident warps); without it the loads are issued at use and latency is hidden by occupancy alone.
template <class Fq, bool PF>
B2M_HD void aff_level_thread(const AffLevel<Fq>& A, const Affine<Fq>* base, uint32_t t) {
  const uint32_t total = B2M_AFF_LDG32(A.off_out + A.B);
  const AffMap mp = aff_map(A, t, total);
  if (!mp.cnt) return;
  const uint32_t cnt = mp.cnt;
  const size_t nth = A.nthreads;
  const uint4* meta = A.meta + t;
  Fq* pref = A.pref + t;
  // ---- pass 1: denominators, running product ----------------------------------------------------
  Fq run = Fq::one();
  {
    uint4 m = meta[0];
    uint4 m1 = cnt > 1 ? meta[nth] : m;
    Fq x1, x2;
    if (PF) {
      x1 = aff_ldx(base, m.x);
      x2 = aff_ldx(base, m.y);
    }
    for (uint32_t k = 0; k < cnt; k++) {
      const uint4 mc = m;
      Fq c1, c2;
      if (PF) {
        c1 = x1;
        c2 = x2;
      } else {
        c1 = aff_ldx(base, mc.x);
        c2 = aff_ldx(base, mc.y);
      }
      if (k + 1 < cnt) {  // the plan runs two outputs ahead, (PF) the operands one
        m = m1;
        if (k + 2 < cnt) m1 = meta[(size_t)(k + 2) * nth];
        if (PF) {
          x1 = aff_ldx(base, m.x);
          x2 = aff_ldx(base, m.y);
        }
      }
      Fq den = Fq::one();
      if (mc.w) {
        if (c1.is_zero() || c2.is_zero() || c1 == c2) {  // rare: infinity, doubling or cancellation
          Fq d;
          const AffKind kind = aff_classify(aff_signed(aff_ld(base, mc.x), mc.x), aff_signed(aff_ld(base, mc.y), mc.y), &d);
          if (kind == AFF_ADD || kind == AFF_DBL) den = d;
        } else {
          den = c2 - c1;
        }
      }
      run = k ? run * den : den;
      B2M_AFF_ST(pref + (size_t)k * nth, run);
    }
  }
  // ---- one inversion per thread (the product of non-zero denominators is never zero) ---------------------
  Fq inv = run.inverse_fast();
  // ---- pass 2: walk back, peel one denominator at a time ----------------------------------------------
  {
    uint4 m = meta[(size_t)(cnt - 1) * nth];
    uint4 m1 = cnt > 1 ? meta[(size_t)(cnt - 2) * nth] : m;
    Affine<Fq> Pn, Qn;
    Fq pfn = run;  // product of the denominators before the output (read for k > 0 only)
    if (PF) {
      Pn = aff_ld(base, m.x);
      Qn = aff_ld(base, m.y);
      if (cnt > 1) pfn = B2M_AFF_LD(pref + (size_t)(cnt - 2) * nth);
    }
    for (uint32_t k = cnt; k-- > 0;) {
      const uint4 mc = m;
      Affine<Fq> P, Q;
      Fq pf = run;
      if (PF) {
        P = Pn;
        Q = Qn;
        pf = pfn;
      } else {
        P = aff_ld(base, mc.x);
        Q = aff_ld(base, mc.y);
        if (k > 0) pf = B2M_AFF_LD(pref + (size_t)(k - 1) * nth);
      }
      P = aff_signed(P, mc.x);
      Q = aff_signed(Q, mc.y);
      if (k > 0) {
        m = m1;
        if (k > 1) m1 = meta[(size_t)(k - 2) * nth];
        if (PF) {
          Pn = aff_ld(base, m.x);
          Qn = aff_ld(base, m.y);
          if (k > 1) pfn = B2M_AFF_LD(pref + (size_t)(k - 2) * nth);
        }
      }
      Affine<Fq> R = P;
      if (mc.w) {
        Fq den;
        const AffKind kind = aff_classify(P, Q, &den);
        if (kind == AFF_COPY_Q) {
          R = Q;
        } else if (kind == AFF_INF) {
          R = Affine<Fq>::inf();
        } else if (kind != AFF_COPY_P) {
          Fq dinv = inv;
          if (k > 0) dinv = inv * pf;
          inv = inv * den;
          Fq lam;
          if (kind == AFF_ADD) {
            lam = (Q.y - P.y) * dinv;
            R.x = lam.sqr() - P.x - Q.x;
          } else {
            const Fq xx = P.x.sqr();
            lam = (xx.dbl() + xx) * dinv;
            R.x = lam.sqr() - P.x.dbl();
          }
          R.y = lam * (P.x - R.x) - P.y;
        }
      }
      const uint32_t o = mp.o0 + k * mp.step;
      B2M_AFF_ST(&A.out[o].x, R.x);
      B2M_AFF_ST(&A.out[o].y, R.y);
      if (A.out_refs) {
        uint2 r;
        r.x = o;
        r.y = mc.z;  // window 0: `out` is addressed directly
        A.out_refs[o] = r;
      }
    }
  }
}

// one output given the inverse of its denominator; returns the denominator (one() if the output needs none)
template <class Fq>
B2M_HD Affine<Fq> aff_finish(const Affine<Fq>& P, const Affine<Fq>& Q, bool pair, const Fq& dinv, Fq* den_out) {
  *den_out = Fq::one();
  if (!pair) return P;
  Fq den;
  const AffKind kind = aff_classify(P, Q, &den);
  if (kind == AFF_COPY_P) return P;
  if (kind == AFF_COPY_Q) return Q;
  if (kind == AFF_INF) return Affine<Fq>::inf();
  *den_out = den;
  Fq lam;
  Affine<Fq> R;
  if (kind == AFF_ADD) {
    lam = (Q.y - P.y) * dinv;
    R.x = lam.sqr() - P.x - Q.x;
  } else {
    const Fq xx = P.x.sqr();
    lam = (xx.dbl() + xx) * dinv;
    R.x = lam.sqr() - P.x.dbl();
  }
  R.y = lam * (P.x - R.x) - P.y;
  return R;
}
template <class Fq>
B2M_HD void aff_store_out(const AffLevel<Fq>& A, uint32_t o, const Affine<Fq>& R, uint32_t bucket) {
  B2M_AFF_ST(&A.out[o].x, R.x);
  B2M_AFF_ST(&A.out[o].y, R.y);
  if (A.out_refs) {
    uint2 r;
    r.x = o;
    r.y = bucket;
    A.out_refs[o] = r;
  }
}

// ---- software-pipelined variant (kernel variants 8 / 9) ---------------------------------------------------------------
// Profiles of the variants above show no saturated pipe -- every warp simply
// runs at its own latency-bound pace (a serial chain of five multiplications per output, each multiplication two carry
// chains, operand loads issued at their point of use), and extra work of ANY kind (more inversions, more loads) adds its full
// time.  This variant restructures the per-thread code instead of relying on co-resident warps:
//  * branch-free fast path: den = fast ? x2 - x1 : 1 with fast = "a plain addition of two finite points with different x"
//    (the same predicate in both passes); everything else -- copies of an unpaired point, P + (-P), doublings, operands at
//    infinity -- takes its denominator out of the shared chain (den = 1) and is recomputed on its own in a cold fix-up,
//    so each loop body is ONE basic block the scheduler can interleave freely;
//  * the addition pass is software-pipelined over the outputs: iteration k peels the denominator of output k
//    (dinv_k = inv * pref_k, inv *= den_k: two independent multiplications) while it finishes output k + 1
//    (lambda, lambda^2, y3: a chain of three) -- two independent instruction streams per warp, and the operands of output
//    k are requested one full iteration before their y coordinates are needed;
//  * exclusive prefix products (pref_k = den_0 ... den_(k-1)), so no first-element special case.
template <class Fq>
B2M_HD bool aff_fast(uint32_t w, const Fq& x1, const Fq& x2) {
  return w != 0 && !x1.is_zero() && !x2.is_zero() && !(x1 == x2);
}
// P + Q for the outputs outside the fast path (own inversion; rare or cheap)
template <class Fq>
B2M_HD Affine<Fq> aff_add_slow(const Affine<Fq>& P, const Affine<Fq>& Q, uint32_t w) {
  if (!w) return P;
  Fq den;
  const AffKind kind = aff_classify(P, Q, &den);
  if (kind == AFF_COPY_P) return P;
  if (kind == AFF_COPY_Q) return Q;
  if (kind == AFF_INF) return Affine<Fq>::inf();
  Fq dummy;
  return aff_finish(P, Q, true, den.inverse_fast(), &dummy);
}

// PHASE 0: both passes in one call.  PHASE 1 / 2: the split form -- two kernels per level.  What limits the fused kernel:
// a single warp can issue a wide multiply only every few cycles (the carry chains), so the multiplier pipe is full only
// while >= 2 warps of a sub-partition are inside multiplication code at the same time; the fused kernel's warps spend
// much of their time elsewhere (operand latency of the denominator pass, the ALU-only inversion) at 2-4 resident warps
// per sub-partition.  Split:
//   PHASE 1 = denominator pass + inversion: ~90 registers, 5-6 CTAs/SM -- the gathers' latency and the inversions'
//             tens of thousands of ALU instructions are spread over 5-6 warps per sub-partition instead of blocking a 128-168-register warp;
//   PHASE 2 = addition pass only: every resident warp is inside multiplication code nearly all the time.
// The chain inverse crosses in A.inv[t].
//   PHASE 3 = denominator pass WITHOUT the inversion: the chain product goes to A.inv[t] and a separate kernel
//             (msm_impl.cuh fq_batch_inverse_kernel) inverts all chain products of the level together -- a second level of
//             Montgomery's trick across threads: one binary-Euclid inversion per 128 chains (8 192 additions) instead of one per
//             chain, executed by one lane while the scan multiplications around it are warp-wide.
template <class Fq, int PHASE, bool PIPE = true>
B2M_HD void aff_level_thread_sp(const AffLevel<Fq>& A, const Affine<Fq>* base, uint32_t t) {
  const uint32_t total = B2M_AFF_LDG32(A.off_out + A.B);
  const AffMap mp = aff_map(A, t, total);
  if (!mp.cnt) {
    if (PHASE == 3) B2M_AFF_ST(A.inv + t, Fq::one());  // (the batch inversion reads every slot)
    return;
  }
  const uint32_t cnt = mp.cnt;
  const size_t nth = A.nthreads;
  const uint4* meta = A.meta + t;
  Fq* pref = A.pref + t;
  Fq inv;
  if (PHASE != 2) {
    // ---- pass 1: exclusive prefix products of the denominators; the plan two outputs ahead, the operands one ---------
    Fq run = Fq::one();
    uint4 m = meta[0];
    uint4 m1 = cnt > 1 ? meta[nth] : m;
    Fq x1 = aff_ldx(base, m.x), x2 = aff_ldx(base, m.y);
    for (uint32_t k = 0; k < cnt; k++) {
      const uint32_t w = m.w;
      const Fq c1 = x1, c2 = x2;
      if (k + 1 < cnt) {
        m = m1;
        if (k + 2 < cnt) m1 = meta[(size_t)(k + 2) * nth];
        x1 = aff_ldx(base, m.x);
        x2 = aff_ldx(base, m.y);
      }
      const Fq d = c2 - c1;
      const Fq den = aff_fast(w, c1, c2) ? d : Fq::one();
      B2M_AFF_ST(pref + (size_t)k * nth, run);
      run = run * den;
    }
    if (PHASE == 3) {
      B2M_AFF_ST(A.inv + t, run);
      return;
    }
    inv = run.inverse_fast();
    if (PHASE == 1) {
      B2M_AFF_ST(A.inv + t, inv);
      return;
    }
  } else {
    inv = B2M_AFF_LD(A.inv + t);
  }
  if (!PIPE) {
    // ---- pass 2, plain form (fewer live registers: more resident warps): one output per iteration -----------------------
    uint4 m = meta[(size_t)(cnt - 1) * nth];
    for (uint32_t k = cnt; k-- > 0;) {
      const uint4 mc = m;
      const Affine<Fq> P = aff_signed(aff_ld(base, mc.x), mc.x), Q = aff_signed(aff_ld(base, mc.y), mc.y);
      const Fq pf = B2M_AFF_LD(pref + (size_t)k * nth);
      if (k > 0) m = meta[(size_t)(k - 1) * nth];
      const bool fast = aff_fast(mc.w, P.x, Q.x);
      const Fq d = Q.x - P.x;
      const Fq den = fast ? d : Fq::one();
      const Fq dinv = inv * pf;
      inv = inv * den;
      const Fq lam = (Q.y - P.y) * dinv;
      Affine<Fq> R;
      R.x = lam.sqr() - P.x - Q.x;
      R.y = lam * (P.x - R.x) - P.y;
      if (!fast) R = aff_add_slow(P, Q, mc.w);  // cold
      aff_store_out(A, mp.o0 + k * mp.step, R, mc.z);
    }
    return;
  }
  // ---- pass 2, software-pipelined -----------------------------------------------------------------------------------
  // current = the output whose denominator has been peeled (dinv_c known) and whose sum is still to be formed
  uint4 m_c = meta[(size_t)(cnt - 1) * nth];
  Affine<Fq> P_c = aff_signed(aff_ld(base, m_c.x), m_c.x), Q_c = aff_signed(aff_ld(base, m_c.y), m_c.y);
  bool fast_c = aff_fast(m_c.w, P_c.x, Q_c.x);
  Fq dinv_c;
  {
    const Fq pf = B2M_AFF_LD(pref + (size_t)(cnt - 1) * nth);
    const Fq d = Q_c.x - P_c.x;
    const Fq den = fast_c ? d : Fq::one();
    dinv_c = inv * pf;
    inv = inv * den;
  }
  for (uint32_t k = cnt - 1; k-- > 0;) {
    // request output k's operands; finish output k + 1 meanwhile
    const uint4 m_n = meta[(size_t)k * nth];
    const Affine<Fq> P_r = aff_ld(base, m_n.x), Q_r = aff_ld(base, m_n.y);
    const Fq pf = B2M_AFF_LD(pref + (size_t)k * nth);
    // stage B (output k + 1): lambda, x3, y3 -- computed unconditionally, replaced below when the output is not a fast one
    const Fq lam = (Q_c.y - P_c.y) * dinv_c;
    Affine<Fq> R;
    R.x = lam.sqr() - P_c.x - Q_c.x;
    R.y = lam * (P_c.x - R.x) - P_c.y;
    // stage A (output k): peel its denominator
    const Affine<Fq> P_n = aff_signed(P_r, m_n.x), Q_n = aff_signed(Q_r, m_n.y);
    const bool fast_n = aff_fast(m_n.w, P_n.x, Q_n.x);
    const Fq d = Q_n.x - P_n.x;
    const Fq den = fast_n ? d : Fq::one();
    const Fq dinv_n = inv * pf;
    inv = inv * den;
    if (!fast_c) R = aff_add_slow(P_c, Q_c, m_c.w);  // cold
    aff_store_out(A, mp.o0 + (k + 1) * mp.step, R, m_c.z);
    m_c = m_n;
    P_c = P_n;
    Q_c = Q_n;
    fast_c = fast_n;
    dinv_c = dinv_n;
  }
  {  // epilogue: output 0
    const Fq lam = (Q_c.y - P_c.y) * dinv_c;
    Affine<Fq> R;
    R.x = lam.sqr() - P_c.x - Q_c.x;
    R.y = lam * (P_c.x - R.x) - P_c.y;
    if (!fast_c) R = aff_add_slow(P_c, Q_c, m_c.w);
    aff_store_out(A, mp.o0, R, m_c.z);
  }
}

}  // namespace b2m
