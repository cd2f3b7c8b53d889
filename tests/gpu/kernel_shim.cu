// Test-only C ABI over the product's device code (marlin_b200/csrc): every entry point uploads host arrays,
// runs the product's own kernel or host driver on one Ctx, and downloads the result, so that
// tests/test_device_kernels_gpu.py can compare single kernels with Python integers at their edge cases.
// Nothing here is part of libb2m.so or include/b2m.h; the headers are included, not copied, and the library is
// compiled with the product's NVFLAGS (tests/gpu/Makefile).
//
// Field ids: 0 = BLS12-381 Fr, 1 = BLS12-381 Fq, 2 = BN254 Fr, 3 = BN254 Fq.  Curve ids: 0 = BLS12-381, 1 = BN254.
// Field elements are little-endian u32 limbs in Montgomery form unless an op says otherwise.
#include "../../marlin_b200/csrc/common.cuh"
#include "../../marlin_b200/csrc/devmem.cuh"
#include "../../marlin_b200/csrc/curve.cuh"
#include "../../marlin_b200/csrc/poly_impl.cuh"
#include "../../marlin_b200/csrc/scan.cuh"

#include <algorithm>
#include <cstring>
#include <string>

using namespace b2m;

namespace {

Ctx* g_ctx = nullptr;
std::string g_err;

template <class Fn>
int guarded(Fn&& fn) {
  try {
    B2M_REQUIRE(g_ctx, B2M_ERR_INVALID_ARG, "kt_ctx_create has not been called");
    fn(*g_ctx);
    return 0;
  } catch (const Error& e) {
    g_err = e.what();
    return e.code;
  } catch (const std::exception& e) {
    g_err = e.what();
    return B2M_ERR_CUDA;
  }
}

// ---- field arithmetic, one element per thread ----------------------------------------------------
// op codes 0-7 are those of tests/host/field_host_shim.cpp
enum { OP_MUL, OP_ADD, OP_SUB, OP_NEG, OP_INV, OP_TO_CANON, OP_FROM_CANON, OP_INV_FAST, OP_SQR, OP_DBL, OP_POW_U64, OP_COUNT };

template <class F>
__global__ void field_op_kernel(int op, const F* a, const F* b, size_t n, F* out) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  F x = ld_fr(a + i), y = ld_fr(b + i), z;
  switch (op) {
    case OP_MUL: z = x * y; break;
    case OP_ADD: z = x + y; break;
    case OP_SUB: z = x - y; break;
    case OP_NEG: z = x.neg(); break;
    case OP_INV: z = x.inverse(); break;
    case OP_TO_CANON: z = x.to_canonical(); break;
    case OP_FROM_CANON: z = F::from_canonical(x); break;
    case OP_INV_FAST: z = x.inverse_fast(); break;
    case OP_SQR: z = x.sqr(); break;
    case OP_DBL: z = x.dbl(); break;
    default: z = x.pow_u64((uint64_t)y.l[0] | ((uint64_t)y.l[1] << 32)); break;  // OP_POW_U64: exponent = low 64 bits of b
  }
  st_fr(out + i, z);
}

template <class F>
void field_op(Ctx& cx, int op, const uint32_t* a, const uint32_t* b, size_t n, uint32_t* out) {
  if (n == 0) return;
  DBuf<F> da(cx, n), db(cx, n), dout(cx, n);
  da.upload(reinterpret_cast<const F*>(a), n);
  db.upload(reinterpret_cast<const F*>(b), n);
  field_op_kernel<F><<<div_up(n, 128), 128, 0, cx.stream>>>(op, da.p, db.p, n, dout.p);
  B2M_CHECK_LAUNCH();
  dout.download(reinterpret_cast<F*>(out), n);
}

// ---- XYZZ group law, one case per thread (the host shim's curve_op, on the device) ----------------
// which: 0 = sum of the case's points via add_mixed (with negate flags), 1 = odd / even points summed with add_mixed
// into two XYZZ accumulators, then combined with full additions (doubling and cancellation through `add`),
// 2 = scalar_mul(first point, k).  Every result leaves through to_affine.
template <class Fq>
__global__ void curve_op_kernel(int which, const Affine<Fq>* pts, const uint8_t* neg, int npts, size_t ncases, const uint32_t* k, int klimbs,
                                Affine<Fq>* out) {
  size_t c = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (c >= ncases) return;
  const Affine<Fq>* P = pts + c * npts;
  const uint8_t* ng = neg + c * npts;
  XYZZ<Fq> acc = XYZZ<Fq>::inf();
  if (which == 0) {
    for (int i = 0; i < npts; i++) acc.add_mixed(P[i], ng[i] != 0);
  } else if (which == 1) {
    XYZZ<Fq> a = XYZZ<Fq>::inf(), b = XYZZ<Fq>::inf();
    for (int i = 0; i < npts; i++) {
      if (i & 1) a.add_mixed(P[i], ng[i] != 0);
      else b.add_mixed(P[i], ng[i] != 0);
    }
    a.add(b);
    acc = a;
    acc.add(XYZZ<Fq>::inf());
    XYZZ<Fq> z = XYZZ<Fq>::inf();
    z.add(acc);
    acc = z;
  } else {
    acc = scalar_mul<Fq>(P[0], k + c * klimbs, klimbs);
  }
  out[c] = acc.to_affine();
}

template <class Fq>
void curve_op(Ctx& cx, int which, const uint32_t* pts, const uint8_t* neg, int npts, size_t ncases, const uint32_t* k, int klimbs, uint32_t* out) {
  using Pt = Affine<Fq>;
  B2M_REQUIRE(which >= 0 && which <= 2 && npts >= 1, B2M_ERR_INVALID_ARG, "bad curve op %d / %d points", which, npts);
  B2M_REQUIRE(which != 2 || (k && klimbs >= 1), B2M_ERR_INVALID_ARG, "scalar_mul needs scalars");
  if (ncases == 0) return;
  const size_t np = ncases * npts;
  DBuf<Pt> dp(cx, np), dout(cx, ncases);
  DBuf<uint8_t> dn(cx, np);
  DBuf<uint32_t> dk(cx, which == 2 ? ncases * klimbs : 1);
  dp.upload(reinterpret_cast<const Pt*>(pts), np);
  if (neg) dn.upload(neg, np);
  else dn.zero();
  if (which == 2) dk.upload(k, ncases * klimbs);
  curve_op_kernel<Fq><<<div_up(ncases, 64), 64, 0, cx.stream>>>(which, dp.p, dn.p, npts, ncases, dk.p, klimbs, dout.p);
  B2M_CHECK_LAUNCH();
  dout.download(reinterpret_cast<Pt*>(out), ncases);
}

// ---- prover glue (poly_impl.cuh) ---------------------------------------------------------------------
template <class Fr>
void rec_suffix_op(Ctx& cx, const uint32_t* in, size_t n, size_t s, const uint32_t* z, bool mul, bool in_place, uint32_t* out) {
  B2M_REQUIRE(s >= 1, B2M_ERR_INVALID_ARG, "stride must be at least 1");
  if (n == 0) return;
  Fr zz;
  memcpy(zz.l, z, sizeof(zz.l));
  DBuf<Fr> din(cx, n), dout(cx, in_place ? 1 : n);
  din.upload(reinterpret_cast<const Fr*>(in), n);
  Fr* dst = in_place ? din.p : dout.p;
  rec_suffix<Fr>(cx, din.p, dst, n, s, zz, mul);
  B2M_CUDA(cudaMemcpyAsync(out, dst, n * sizeof(Fr), cudaMemcpyDeviceToHost, cx.stream));
  cx.sync();
}

template <class Fr>
void batch_inverse_op(Ctx& cx, uint32_t* data, size_t n) {
  if (n == 0) return;
  DBuf<Fr> d(cx, n);
  d.upload(reinterpret_cast<const Fr*>(data), n);
  batch_inverse<Fr>(cx, d.p, n);
  d.download(reinterpret_cast<Fr*>(data), n);
}

template <class Fr>
void spmv_op(Ctx& cx, const uint32_t* row_ptr, const uint32_t* col, const uint32_t* coeff, const uint32_t* z, size_t nrows, uint32_t* out) {
  if (nrows == 0) return;
  const size_t nnz = row_ptr[nrows];
  size_t nz = 1;
  for (size_t e = 0; e < nnz; e++) nz = std::max(nz, (size_t)col[e] + 1);
  DBuf<uint32_t> drp(cx, nrows + 1), dcol(cx, nnz);
  DBuf<Fr> dcoeff(cx, nnz), dz(cx, nz), dout(cx, nrows);
  drp.upload(row_ptr, nrows + 1);
  if (nnz) {
    dcol.upload(col, nnz);
    dcoeff.upload(reinterpret_cast<const Fr*>(coeff), nnz);
  }
  if (nnz) dz.upload(reinterpret_cast<const Fr*>(z), nz);
  // the prover's launch (prover_impl.cuh, z_A / z_B)
  spmv_kernel<Fr><<<div_up(nrows, 256), 256, 0, cx.stream>>>(drp.p, dcol.p, dcoeff.p, dz.p, nrows, dout.p);
  B2M_CHECK_LAUNCH();
  dout.download(reinterpret_cast<Fr*>(out), nrows);
}

template <class Fr>
void sample_op(Ctx& cx, const uint8_t* key, int rounds, uint64_t pos0, size_t nattempts, uint32_t* cand, uint32_t* accept) {
  if (nattempts == 0) return;
  ChaChaKey k;
  memcpy(k.k, key, 32);
  DBuf<Fr> dc(cx, nattempts);
  DBuf<uint32_t> da(cx, nattempts);
  // the launch of sample_mask (prover_impl.cuh)
  sample_attempts_kernel<Fr><<<div_up(nattempts, 128), 128, 0, cx.stream>>>(k, rounds, pos0, nattempts, dc.p, da.p);
  B2M_CHECK_LAUNCH();
  dc.download(reinterpret_cast<Fr*>(cand), nattempts);
  da.download(accept, nattempts);
}

}  // namespace

extern "C" {

const char* kt_last_error() { return g_err.c_str(); }

int kt_ctx_create(int device) {
  try {
    if (!g_ctx) g_ctx = new Ctx(device);
    return 0;
  } catch (const Error& e) {
    g_err = e.what();
    return e.code;
  }
}

void kt_ctx_destroy() {
  if (g_ctx) {
    cudaStreamSynchronize(g_ctx->stream);
    delete g_ctx;
    g_ctx = nullptr;
  }
}

int kt_field_op(int field, int op, const uint32_t* a, const uint32_t* b, size_t n, uint32_t* out) {
  return guarded([&](Ctx& cx) {
    B2M_REQUIRE(op >= 0 && op < OP_COUNT, B2M_ERR_INVALID_ARG, "unknown field op %d", op);
    switch (field) {
      case 0: field_op<FrBls>(cx, op, a, b, n, out); break;
      case 1: field_op<FqBls>(cx, op, a, b, n, out); break;
      case 2: field_op<FrBn>(cx, op, a, b, n, out); break;
      case 3: field_op<FqBn>(cx, op, a, b, n, out); break;
      default: B2M_REQUIRE(false, B2M_ERR_INVALID_ARG, "unknown field %d", field);
    }
  });
}

int kt_curve_op(int curve, int which, const uint32_t* pts, const uint8_t* neg, int npts, size_t ncases, const uint32_t* k, int klimbs,
                uint32_t* out) {
  return guarded([&](Ctx& cx) {
    if (curve == 0) curve_op<FqBls>(cx, which, pts, neg, npts, ncases, k, klimbs, out);
    else curve_op<FqBn>(cx, which, pts, neg, npts, ncases, k, klimbs, out);
  });
}

int kt_scan_u32(const uint32_t* in, size_t n, uint32_t* out) {
  return guarded([&](Ctx& cx) {
    DBuf<uint32_t> din(cx, n), dout(cx, n);
    if (n) din.upload(in, n);
    exclusive_scan_u32(cx, din.p, dout.p, n);
    if (n) dout.download(out, n);
    cx.sync();
  });
}

int kt_rec_suffix(int curve, const uint32_t* in, size_t n, size_t s, const uint32_t* z, int mul, int in_place, uint32_t* out) {
  return guarded([&](Ctx& cx) {
    if (curve == 0) rec_suffix_op<FrBls>(cx, in, n, s, z, mul != 0, in_place != 0, out);
    else rec_suffix_op<FrBn>(cx, in, n, s, z, mul != 0, in_place != 0, out);
  });
}

int kt_batch_inverse(int curve, uint32_t* data, size_t n) {
  return guarded([&](Ctx& cx) {
    if (curve == 0) batch_inverse_op<FrBls>(cx, data, n);
    else batch_inverse_op<FrBn>(cx, data, n);
  });
}

int kt_spmv(int curve, const uint32_t* row_ptr, const uint32_t* col, const uint32_t* coeff, const uint32_t* z, size_t nrows, uint32_t* out) {
  return guarded([&](Ctx& cx) {
    if (curve == 0) spmv_op<FrBls>(cx, row_ptr, col, coeff, z, nrows, out);
    else spmv_op<FrBn>(cx, row_ptr, col, coeff, z, nrows, out);
  });
}

int kt_sample(int curve, const uint8_t* key, int rounds, uint64_t pos0, size_t nattempts, uint32_t* cand, uint32_t* accept) {
  return guarded([&](Ctx& cx) {
    B2M_REQUIRE(rounds == 8 || rounds == 12 || rounds == 20, B2M_ERR_INVALID_ARG, "ChaCha rounds %d", rounds);
    if (curve == 0) sample_op<FrBls>(cx, key, rounds, pos0, nattempts, cand, accept);
    else sample_op<FrBn>(cx, key, rounds, pos0, nattempts, cand, accept);
  });
}

}  // extern "C"
