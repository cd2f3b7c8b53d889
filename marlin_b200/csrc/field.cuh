// Montgomery prime-field arithmetic for sm_90a, 32-bit limbs, PTX carry chains.
//
// Replaces (for the prover hot path) ark-ff 0.3 `Fp256<P>` / `Fp384<P>`
// [U ark-ff src/fields/models/fp_256.rs, fp_384.rs]: same Montgomery radix
// (R = 2^256 / 2^384), same little-endian limb order, so an `Fp<..>` here is
// byte-identical in memory to arkworks' `[u64; 4]` / `[u64; 6]` representation.
//
// The multiplier keeps the running product split into an "even" and an "odd"
// accumulator (T = E + 2^32*O) so that every 32x32->64 product lands in an aligned
// 64-bit slot and each row is two straight carry chains of mad.lo.cc/madc.hi.cc
// pairs, which ptxas fuses into IMAD.WIDE.U32(.X).  The same source compiles for
// the host (carry flag emulated) so tests/ can check limb-level behaviour without
// a GPU.
#pragma once
#include <cstdint>
#include <cstring>

#ifndef __CUDACC__
#ifndef __host__
#define __host__
#endif
#ifndef __device__
#define __device__
#endif
#ifndef __forceinline__
#ifdef B2M_HOST_LIGHT_INLINE  // host test builds: let the compiler decide (the fully inlined form takes minutes to compile)
#define __forceinline__ inline
#else
#define __forceinline__ inline __attribute__((always_inline))
#endif
#endif
#endif

#include "field_params.h"

#define B2M_HD __host__ __device__ __forceinline__

namespace b2m {

// ---------------------------------------------------------------------------
// carry-chain primitives
// ---------------------------------------------------------------------------
#ifdef __CUDA_ARCH__
__device__ __forceinline__ uint32_t add_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("add.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
__device__ __forceinline__ uint32_t addc_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("addc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
__device__ __forceinline__ uint32_t addc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("addc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
__device__ __forceinline__ uint32_t sub_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("sub.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
__device__ __forceinline__ uint32_t subc_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("subc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
__device__ __forceinline__ uint32_t subc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("subc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
__device__ __forceinline__ uint32_t mad_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("mad.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
__device__ __forceinline__ uint32_t madc_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("madc.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
__device__ __forceinline__ uint32_t madc_hi_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("madc.hi.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
__device__ __forceinline__ uint32_t madc_hi(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("madc.hi.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
#else
// Host emulation of the PTX condition-code flag (CC.CF); one flag per thread.
inline uint32_t& cc_flag() { static thread_local uint32_t cf = 0; return cf; }
inline uint32_t add_cc(uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a + b; cc_flag() = (uint32_t)(t >> 32); return (uint32_t)t; }
inline uint32_t addc_cc(uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a + b + cc_flag(); cc_flag() = (uint32_t)(t >> 32); return (uint32_t)t; }
inline uint32_t addc(uint32_t a, uint32_t b) { return a + b + cc_flag(); }
inline uint32_t sub_cc(uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a - b; cc_flag() = (uint32_t)(t >> 63); return (uint32_t)t; }
inline uint32_t subc_cc(uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a - b - cc_flag(); cc_flag() = (uint32_t)(t >> 63); return (uint32_t)t; }
inline uint32_t subc(uint32_t a, uint32_t b) { return a - b - cc_flag(); }
inline uint32_t mad_lo_cc(uint32_t a, uint32_t b, uint32_t c) { return add_cc((uint32_t)((uint64_t)a * b), c); }
inline uint32_t madc_lo_cc(uint32_t a, uint32_t b, uint32_t c) { return addc_cc((uint32_t)((uint64_t)a * b), c); }
inline uint32_t madc_hi_cc(uint32_t a, uint32_t b, uint32_t c) { return addc_cc((uint32_t)(((uint64_t)a * b) >> 32), c); }
inline uint32_t madc_hi(uint32_t a, uint32_t b, uint32_t c) { return addc((uint32_t)(((uint64_t)a * b) >> 32), c); }
#endif

// acc[2k], acc[2k+1] = a[2k] * b  (a is read with stride 2 starting at a[0]).
template <int N>
B2M_HD void mul_n(uint32_t* acc, const uint32_t* a, uint32_t b) {
#pragma unroll
  for (int k = 0; k < N; k += 2) {
    uint64_t w = (uint64_t)a[k] * b;
    acc[k] = (uint32_t)w;
    acc[k + 1] = (uint32_t)(w >> 32);
  }
}

// acc += sum_k a[2k]*b*2^(64k); leaves the carry-out in CC.CF.
template <int N>
B2M_HD void cmad_n(uint32_t* acc, const uint32_t* a, uint32_t b) {
  acc[0] = mad_lo_cc(a[0], b, acc[0]);
  acc[1] = madc_hi_cc(a[0], b, acc[1]);
#pragma unroll
  for (int k = 2; k < N; k += 2) {
    acc[k] = madc_lo_cc(a[k], b, acc[k]);
    acc[k + 1] = madc_hi_cc(a[k], b, acc[k + 1]);
  }
}

// acc = (acc >> 64) + sum_k a[2k]*b*2^(64k) + CC.CF   (no carry-out possible).
template <int N>
B2M_HD void madc_n_rshift(uint32_t* acc, const uint32_t* a, uint32_t b) {
#pragma unroll
  for (int k = 0; k < N - 2; k += 2) {
    acc[k] = madc_lo_cc(a[k], b, acc[k + 2]);
    acc[k + 1] = madc_hi_cc(a[k], b, acc[k + 3]);
  }
  acc[N - 2] = madc_lo_cc(a[N - 2], b, 0u);
  acc[N - 1] = madc_hi(a[N - 2], b, 0u);
}

template <class P>
struct Fp {
  using Params = P;
  static constexpr int N = P::N;
  uint32_t l[N];

  B2M_HD static Fp zero() {
    Fp r;
#pragma unroll
    for (int i = 0; i < N; i++) r.l[i] = 0;
    return r;
  }
  B2M_HD static Fp one() {  // Montgomery form of 1
    Fp r;
#pragma unroll
    for (int i = 0; i < N; i++) r.l[i] = P::r(i);
    return r;
  }
  B2M_HD static Fp modulus() {
    Fp r;
#pragma unroll
    for (int i = 0; i < N; i++) r.l[i] = P::mod(i);
    return r;
  }
  B2M_HD static Fp r2() {
    Fp r;
#pragma unroll
    for (int i = 0; i < N; i++) r.l[i] = P::r2(i);
    return r;
  }
  B2M_HD bool is_zero() const {
    uint32_t t = 0;
#pragma unroll
    for (int i = 0; i < N; i++) t |= l[i];
    return t == 0;
  }
  B2M_HD bool operator==(const Fp& o) const {
    uint32_t t = 0;
#pragma unroll
    for (int i = 0; i < N; i++) t |= l[i] ^ o.l[i];
    return t == 0;
  }
  B2M_HD bool operator!=(const Fp& o) const { return !(*this == o); }

  // r = a + b mod p  (inputs < p)
  B2M_HD friend Fp operator+(const Fp& a, const Fp& b) {
    Fp r, t;
    r.l[0] = add_cc(a.l[0], b.l[0]);
#pragma unroll
    for (int i = 1; i < N - 1; i++) r.l[i] = addc_cc(a.l[i], b.l[i]);
    r.l[N - 1] = addc(a.l[N - 1], b.l[N - 1]);  // p < 2^(32N-1): no carry out
    t.l[0] = sub_cc(r.l[0], P::mod(0));
#pragma unroll
    for (int i = 1; i < N; i++) t.l[i] = subc_cc(r.l[i], P::mod(i));
    uint32_t borrow = subc(0u, 0u);  // 0xffffffff if r < p
#pragma unroll
    for (int i = 0; i < N; i++) r.l[i] = borrow ? r.l[i] : t.l[i];
    return r;
  }
  B2M_HD friend Fp operator-(const Fp& a, const Fp& b) {
    Fp r;
    r.l[0] = sub_cc(a.l[0], b.l[0]);
#pragma unroll
    for (int i = 1; i < N; i++) r.l[i] = subc_cc(a.l[i], b.l[i]);
    uint32_t borrow = subc(0u, 0u);
    r.l[0] = add_cc(r.l[0], P::mod(0) & borrow);
#pragma unroll
    for (int i = 1; i < N - 1; i++) r.l[i] = addc_cc(r.l[i], P::mod(i) & borrow);
    r.l[N - 1] = addc(r.l[N - 1], P::mod(N - 1) & borrow);
    return r;
  }
  B2M_HD Fp neg() const { return is_zero() ? *this : (modulus_raw_sub(*this)); }
  B2M_HD static Fp modulus_raw_sub(const Fp& a) {
    Fp r;
    r.l[0] = sub_cc(P::mod(0), a.l[0]);
#pragma unroll
    for (int i = 1; i < N - 1; i++) r.l[i] = subc_cc(P::mod(i), a.l[i]);
    r.l[N - 1] = subc(P::mod(N - 1), a.l[N - 1]);
    return r;
  }
  B2M_HD Fp dbl() const { return *this + *this; }

  // Montgomery product a*b*R^-1 mod p.
  B2M_HD friend Fp operator*(const Fp& a, const Fp& b) {
    uint32_t ev[N], od[N];
    uint32_t mod_[N];
#pragma unroll
    for (int i = 0; i < N; i++) mod_[i] = P::mod(i);
#pragma unroll
    for (int i = 0; i < N; i += 2) {
      row(ev, od, a.l, b.l[i], mod_, i == 0);
      row(od, ev, a.l, b.l[i + 1], mod_, false);
    }
    // pending division by 2^32: R[j] = ev[j] + od[j+1]
    Fp r;
    r.l[0] = add_cc(ev[0], od[1]);
#pragma unroll
    for (int i = 1; i < N - 1; i++) r.l[i] = addc_cc(ev[i], od[i + 1]);
    r.l[N - 1] = addc(ev[N - 1], 0u);
    return r.reduce_once();
  }
  B2M_HD Fp sqr() const { return (*this) * (*this); }

  // one CIOS row: E-role array `e`, O-role array `o`  (T = e + 2^32 * o).
  B2M_HD static void row(uint32_t* e, uint32_t* o, const uint32_t* a, uint32_t bi, const uint32_t* mod_, bool first) {
    if (first) {
      mul_n<N>(o, a + 1, bi);
      mul_n<N>(e, a, bi);
    } else {
      // T/2^32: new E = old O + old E[1]; new O = old E >> 64.  Here `e` is the old O array.
      e[0] = add_cc(e[0], o[1]);
      madc_n_rshift<N>(o, a + 1, bi);
      cmad_n<N>(e, a, bi);
      o[N - 1] = addc(o[N - 1], 0u);
    }
    uint32_t m = e[0] * P::NINV;
    cmad_n<N>(o, mod_ + 1, m);  // carry-out is provably zero (T < 2^(32(N+1)))
    cmad_n<N>(e, mod_, m);
    o[N - 1] = addc(o[N - 1], 0u);
  }

  B2M_HD Fp reduce_once() const {
    Fp t, r;
    t.l[0] = sub_cc(l[0], P::mod(0));
#pragma unroll
    for (int i = 1; i < N; i++) t.l[i] = subc_cc(l[i], P::mod(i));
    uint32_t borrow = subc(0u, 0u);
#pragma unroll
    for (int i = 0; i < N; i++) r.l[i] = borrow ? l[i] : t.l[i];
    return r;
  }

  // Montgomery -> canonical integer (little-endian limbs), i.e. ark-ff `into_repr()`.
  B2M_HD Fp to_canonical() const {
    Fp o = zero();
    o.l[0] = 1;
    return (*this) * o;
  }
  // canonical integer (< p) -> Montgomery, i.e. ark-ff `from_repr()`.
  B2M_HD static Fp from_canonical(const Fp& c) { return c * r2(); }
  B2M_HD static Fp from_u64(uint64_t v) {
    Fp c = zero();
    c.l[0] = (uint32_t)v;
    c.l[1] = (uint32_t)(v >> 32);
    return from_canonical(c);
  }

  // x^e for a little-endian limb exponent (square-and-multiply, MSB first).
  B2M_HD Fp pow_limbs(const uint32_t* e, int nlimbs) const {
    Fp r = one();
    bool started = false;
    for (int i = nlimbs - 1; i >= 0; i--) {
      for (int b = 31; b >= 0; b--) {
        if (started) r = r.sqr();
        if ((e[i] >> b) & 1u) {
          r = started ? r * (*this) : *this;
          started = true;
        }
      }
    }
    return r;
  }
  B2M_HD Fp pow_u64(uint64_t e) const {
    uint32_t ee[2] = {(uint32_t)e, (uint32_t)(e >> 32)};
    return pow_limbs(ee, 2);
  }
  // Fermat inverse x^(p-2); inverse(0) = 0.
  B2M_HD Fp inverse() const {
    uint32_t e[N];
#pragma unroll
    for (int i = 0; i < N; i++) e[i] = P::pm2(i);
    return pow_limbs(e, N);
  }
  // Inverse by the binary extended Euclid (Kaliski's almost-inverse, shifts batched by trailing-zero count):
  // ~270 subtract-and-shift steps of plain limb adds / shifts -- an order of magnitude fewer issue slots than
  // the Fermat ladder and none of them on the multiplier pipe, so in a kernel whose other warps are busy
  // multiplying it is nearly free.  Data-dependent trip count (NOT constant time; nothing here is secret to
  // the GPU).  inverse_fast(0) = 0.
  B2M_HD Fp inverse_fast() const {
    if (is_zero()) return *this;
    // With x = the limbs of *this read as an integer, the loop keeps (mod p)
    //   x * ra = -sg * a * 2^k,   x * rb = sg * b * 2^k,   a * rb + b * ra = p   (so ra, rb <= p: no overflow)
    // and ends with a == b == gcd = 1, i.e. x^-1 * 2^k = sg * rb.
    uint32_t a[N], b[N], ra[N], rb[N];
#pragma unroll
    for (int i = 0; i < N; i++) {
      a[i] = P::mod(i);
      b[i] = l[i];
      ra[i] = 0;
      rb[i] = 0;
    }
    rb[0] = 1;
    uint32_t k = 0;
    bool negate = false;
    while (!(b[0] & 1u)) {  // x even: halve b (ra = 0 needs no doubling)
      uint32_t z = b[0] ? ctz32(b[0]) : 31u;
      shr_limbs(b, z);
      k += z;
    }
    for (;;) {
      // a, b odd
      uint32_t t[N];
      t[0] = sub_cc(a[0], b[0]);
#pragma unroll
      for (int i = 1; i < N; i++) t[i] = subc_cc(a[i], b[i]);
      uint32_t borrow = subc(0u, 0u);
      uint32_t nz = 0;
#pragma unroll
      for (int i = 0; i < N; i++) nz |= t[i];
      if (nz == 0) break;
      if (borrow) {  // a < b: swap the two (value, cofactor) pairs, flip the sign
        negate = !negate;
        uint32_t c = 1u;  // a <- b - a = -t
#pragma unroll
        for (int i = 0; i < N; i++) {
          uint32_t v = ~t[i] + c;
          c = (c && v == 0) ? 1u : 0u;
          t[i] = v;
          uint32_t w = ra[i];
          ra[i] = rb[i];
          rb[i] = w;
          b[i] = a[i];
        }
      }
#pragma unroll
      for (int i = 0; i < N; i++) a[i] = t[i];
      ra[0] = add_cc(ra[0], rb[0]);
#pragma unroll
      for (int i = 1; i < N - 1; i++) ra[i] = addc_cc(ra[i], rb[i]);
      ra[N - 1] = addc(ra[N - 1], rb[N - 1]);
      do {  // a even and non-zero
        uint32_t z = a[0] ? ctz32(a[0]) : 31u;
        shr_limbs(a, z);
        shl_limbs(rb, z);
        k += z;
      } while (!(a[0] & 1u));
    }
    Fp y;
#pragma unroll
    for (int i = 0; i < N; i++) y.l[i] = rb[i];
    if (negate) y = modulus_raw_sub(y);
    // y = x^-1 * 2^k with x = v * R  =>  v^-1 * R = x^-1 * R^2 = y * 2^(64 N - k)
    uint32_t e = 64u * N - k;
    uint32_t extra = e > 32u * N - 1 ? e - (32u * N - 1) : 0u;
    e -= extra;
    Fp pw = zero();
    pw.l[e >> 5] = 1u << (e & 31u);
    y = (y * r2()) * pw;  // (y * R) * 2^e / R
    for (uint32_t i = 0; i < extra; i++) y = y.dbl();
    return y;
  }
  B2M_HD static uint32_t ctz32(uint32_t v) {
#ifdef __CUDA_ARCH__
    return (uint32_t)(__ffs((int)v) - 1);
#else
    return (uint32_t)__builtin_ctz(v);
#endif
  }
  B2M_HD static void shr_limbs(uint32_t* v, uint32_t z) {  // 1 <= z <= 31
#pragma unroll
    for (int i = 0; i < N - 1; i++) v[i] = (v[i] >> z) | (v[i + 1] << (32u - z));
    v[N - 1] >>= z;
  }
  B2M_HD static void shl_limbs(uint32_t* v, uint32_t z) {  // 1 <= z <= 31
#pragma unroll
    for (int i = N - 1; i > 0; i--) v[i] = (v[i] << z) | (v[i - 1] >> (32u - z));
    v[0] <<= z;
  }
  // canonical value > (p-1)/2 ?  (`self > -self` in ark-ec's y-sign flag)  -- input is canonical.
  B2M_HD bool canonical_gt_half() const {
    for (int i = N - 1; i >= 0; i--) {
      uint32_t h = P::half(i);
      if (l[i] != h) return l[i] > h;
    }
    return false;
  }
};

using FrBls = Fp<BlsFrParams>;
using FqBls = Fp<BlsFqParams>;
using FrBn = Fp<BnFrParams>;
using FqBn = Fp<BnFqParams>;
using FrBls377 = Fp<Bls377FrParams>;
using FqBls377 = Fp<Bls377FqParams>;

}  // namespace b2m
