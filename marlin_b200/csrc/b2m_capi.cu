// extern "C" boundary of libb2m.so (declared in include/b2m.h).  Level 0: NTT / MSM / SRS.
// The prover-level entry points live in prover.cu.
#include "capi_types.cuh"
#include "prover.cuh"
#include "verify.cuh"
#include "comm.cuh"
#include <algorithm>
#include "g2_host.hpp"
#include "ark_points.cuh"
#include "g2_decode.cuh"
#include "circom.cuh"

namespace b2m {
thread_local std::string g_last_error;
}

using namespace b2m;

extern "C" {

const char* b2m_last_error(void) { return g_last_error.c_str(); }
const char* b2m_version(void) { return "b2m 0.1 (sm_90a)"; }

int b2m_ctx_create(int device, b2m_ctx** out) {
  return guard([&] {
    B2M_REQUIRE(out != nullptr, B2M_ERR_INVALID_ARG, "out is null");
    *out = new b2m_ctx(device);
  });
}

void b2m_ctx_destroy(b2m_ctx* ctx) {
  if (!ctx) return;
  if (ctx->children > 0) {  // SRSs still borrow this context: freed with the last of them
    ctx->dead = true;
    return;
  }
  b2m_release_ctx(ctx);
}

unsigned long long b2m_ctx_launches(const b2m_ctx* ctx) { return ctx ? ctx->cx.launches : 0; }

int b2m_ctx_set_memory_limit(b2m_ctx* ctx, size_t bytes) {
  return guard([&] {
    B2M_REQUIRE(ctx != nullptr, B2M_ERR_INVALID_ARG, "null argument");
    ctx->cx.memory_limit = bytes;
  });
}

int b2m_ctx_memory(b2m_ctx* ctx, size_t* out) {
  return guard([&] {
    B2M_REQUIRE(ctx && out, B2M_ERR_INVALID_ARG, "null argument");
    Ctx& cx = ctx->cx;
    cx.use();
    cx.sync();
    out[0] = (size_t)cx.pool_attr(cudaMemPoolAttrUsedMemCurrent);
    out[1] = (size_t)cx.pool_attr(cudaMemPoolAttrUsedMemHigh);
    out[2] = (size_t)cx.pool_attr(cudaMemPoolAttrReservedMemCurrent);
    uint64_t zero = 0;  // the high-water mark restarts from what is in use now
    B2M_CUDA(cudaMemPoolSetAttribute(cx.pool, cudaMemPoolAttrUsedMemHigh, &zero));
  });
}

int b2m_comm_unique_id(uint8_t* id, size_t cap) {
  return guard([&] {
    B2M_REQUIRE(id && cap >= sizeof(ncclUniqueId), B2M_ERR_INVALID_ARG, "id buffer must hold %zu bytes", sizeof(ncclUniqueId));
    ncclUniqueId u;
    B2M_NCCL(NcclApi::get().GetUniqueId(&u));
    memcpy(id, &u, sizeof(u));
  });
}

int b2m_ctx_attach_comm(b2m_ctx* ctx, const uint8_t* id, size_t id_len, int rank, int world) {
  return guard([&] {
    B2M_REQUIRE(ctx && id && id_len >= sizeof(ncclUniqueId), B2M_ERR_INVALID_ARG, "bad unique id");
    B2M_REQUIRE(world >= 1 && rank >= 0 && rank < world, B2M_ERR_INVALID_ARG, "bad rank %d / world %d", rank, world);
    ctx->cx.use();
    if (world > 1) {
      ncclUniqueId u;
      memcpy(&u, id, sizeof(u));
      ncclComm_t comm;
      B2M_NCCL(NcclApi::get().CommInitRank(&comm, world, u, rank));
      ctx->cx.comm = comm;
    }
    ctx->cx.rank = rank;
    ctx->cx.world = world;
  });
}

int b2m_ctx_profile(b2m_ctx* ctx, int enable) {
  return guard([&] {
    B2M_REQUIRE(ctx != nullptr, B2M_ERR_INVALID_ARG, "null argument");
    ctx->cx.use();
    if (!enable) ctx->cx.span_report();
    ctx->cx.profiling = enable != 0;
  });
}

int b2m_ctx_profile_report(b2m_ctx* ctx, char* json, size_t cap) {
  return guard([&] {
    B2M_REQUIRE(ctx && json && cap > 0, B2M_ERR_INVALID_ARG, "null argument");
    ctx->cx.use();
    snprintf(json, cap, "%s", ctx->cx.span_report().c_str());
  });
}

int b2m_ntt(b2m_ctx* ctx, int curve, uint64_t* data, unsigned log_n, int inverse, int coset) {
  return guard([&] {
    B2M_REQUIRE(ctx && data, B2M_ERR_INVALID_ARG, "null argument");
    ctx->cx.use();
    with_curve(curve, [&](auto t) { ctx->ntt<typename decltype(t)::Fr>().run_host(data, log_n, inverse != 0, coset != 0); });
  });
}

int b2m_srs_create_layout(b2m_ctx* ctx, int curve, const uint64_t* powers_of_g, size_t n_g, const uint64_t* powers_of_gamma_g,
                          const uint64_t* gamma_indices, size_t n_gamma, int window_bits, int window_tables, b2m_srs** out) {
  return guard([&] {
    B2M_REQUIRE(ctx && powers_of_g && out, B2M_ERR_INVALID_ARG, "null argument");
    require_curve(curve);
    B2M_REQUIRE(window_tables >= 0, B2M_ERR_INVALID_ARG, "window_tables %d < 0", window_tables);
    ctx->cx.use();
    *out = new b2m_srs(ctx, curve, powers_of_g, n_g, powers_of_gamma_g, gamma_indices, n_gamma, window_bits, window_tables);
    ctx->children++;
  });
}

int b2m_srs_create(b2m_ctx* ctx, int curve, const uint64_t* powers_of_g, size_t n_g, const uint64_t* powers_of_gamma_g,
                   const uint64_t* gamma_indices, size_t n_gamma, int window_bits, b2m_srs** out) {
  return b2m_srs_create_layout(ctx, curve, powers_of_g, n_g, powers_of_gamma_g, gamma_indices, n_gamma, window_bits, 0, out);
}

void b2m_srs_destroy(b2m_srs* srs) {
  if (!srs) return;
  if (srs->children > 0) {  // indexes / committer keys still borrow this SRS: freed with the last of them
    srs->dead = true;
    return;
  }
  b2m_release_srs(srs);
}

size_t b2m_srs_size(const b2m_srs* srs) { return srs ? srs->n_g : 0; }
int b2m_srs_window_bits(const b2m_srs* srs) { return srs ? srs->window_bits() : 0; }
int b2m_srs_affine_levels(const b2m_srs* srs) { return srs ? srs->affine_levels() : 0; }
int b2m_srs_window_tables(const b2m_srs* srs) { return srs ? srs->window_tables() : 0; }
int b2m_srs_layout(const b2m_srs* srs, size_t* out) {
  return guard([&] {
    B2M_REQUIRE(srs && out, B2M_ERR_INVALID_ARG, "null argument");
    const MsmBytes& b = srs->layout.bytes;
    const size_t v[8] = {(size_t)srs->window_bits(), (size_t)srs->window_tables(), srs->layout.max_pairs, b.tables, b.circuit, b.msm, b.total(),
                         srs->budget};
    memcpy(out, v, sizeof(v));
  });
}

int b2m_srs_msm(b2m_srs* srs, size_t base_off, const uint64_t* scalars, size_t n, uint64_t* out_xy, int* out_is_inf) {
  return guard([&] {
    B2M_REQUIRE(srs && out_xy && (scalars || n == 0), B2M_ERR_INVALID_ARG, "null argument");
    srs->ctx->cx.use();
    with_curve(srs->curve, [&](auto t) { srs->msm<typename decltype(t)::Fr>()->run_host(base_off, scalars, n, out_xy, out_is_inf); });
  });
}

}  // extern "C"
void b2m_release_ctx(b2m_ctx* ctx) {
  cudaSetDevice(ctx->cx.device);
  cudaStreamSynchronize(ctx->cx.stream);
  if (ctx->cx.comm) NcclApi::get().CommDestroy(static_cast<ncclComm_t>(ctx->cx.comm));
  delete ctx;
}
void b2m_release_srs(b2m_srs* srs) {
  b2m_ctx* ctx = srs->ctx;
  ctx->cx.use();
  cudaStreamSynchronize(ctx->cx.stream);
  delete srs;
  if (--ctx->children == 0 && ctx->dead) b2m_release_ctx(ctx);
}
extern "C" {

int b2m_msm_g1(b2m_ctx* ctx, int curve, const uint64_t* bases_xy, const uint64_t* scalars, size_t n, uint64_t* out_xy,
               int* out_is_inf) {
  b2m_srs* srs = nullptr;
  if (n == 0) {
    if (out_is_inf) *out_is_inf = 1;
    return B2M_OK;
  }
  int rc = b2m_srs_create(ctx, curve, bases_xy, n, nullptr, nullptr, 0, 0, &srs);
  if (rc != B2M_OK) return rc;
  rc = b2m_srs_msm(srs, 0, scalars, n, out_xy, out_is_inf);
  b2m_srs_destroy(srs);
  return rc;
}

int b2m_g1_powers(b2m_ctx* ctx, int curve, const uint64_t* g_xy, const uint64_t* beta, size_t n, uint64_t* out_powers_xy) {
  return guard([&] {
    B2M_REQUIRE(ctx && g_xy && beta && out_powers_xy, B2M_ERR_INVALID_ARG, "null argument");
    ctx->cx.use();
    with_curve(curve, [&](auto t) {
      using Fr = typename decltype(t)::Fr;
      using Fq = typename decltype(t)::Fq;
      Msm<Fr, Fq>::g1_powers_host(ctx->cx, g_xy, beta, n, out_powers_xy);
    });
  });
}

int b2m_fixed_base_msm(b2m_ctx* ctx, int curve, const uint64_t* g_xy, const uint64_t* scalars, size_t n, uint64_t* out_xy) {
  return guard([&] {
    B2M_REQUIRE(ctx && g_xy && (scalars || n == 0) && (out_xy || n == 0), B2M_ERR_INVALID_ARG, "null argument");
    ctx->cx.use();
    with_curve(curve, [&](auto t) {
      using Fr = typename decltype(t)::Fr;
      using Fq = typename decltype(t)::Fq;
      Msm<Fr, Fq>::fixed_base_host(ctx->cx, g_xy, scalars, nullptr, 0, n, out_xy);
    });
  });
}

int b2m_srs_export_g1(b2m_srs* srs, size_t first, size_t n, uint8_t* out) {
  return guard([&] {
    B2M_REQUIRE(srs && (out || n == 0), B2M_ERR_INVALID_ARG, "null argument");
    B2M_REQUIRE(first + n <= srs->n_g, B2M_ERR_INVALID_ARG, "powers [%zu, %zu) of %zu", first, first + n, srs->n_g);
    srs->ctx->cx.use();
    with_curve(srs->curve, [&](auto t) {
      using Fr = typename decltype(t)::Fr;
      using Fq = typename decltype(t)::Fq;
      const auto& m = srs->msm<Fr>();
      B2M_REQUIRE(m->tab_world == 1, B2M_ERR_UNSUPPORTED, "export from a sharded key");
      Msm<Fr, Fq>::g1_to_bytes(srs->ctx->cx, m->tables.p + first, nullptr, n, out);
    });
  });
}
int b2m_g1_to_uncompressed(b2m_ctx* ctx, int curve, const uint64_t* points_xy, size_t n, uint8_t* out) {
  return guard([&] {
    B2M_REQUIRE(ctx && ((points_xy && out) || n == 0), B2M_ERR_INVALID_ARG, "null argument");
    ctx->cx.use();
    with_curve(curve, [&](auto t) {
      using Fr = typename decltype(t)::Fr;
      using Fq = typename decltype(t)::Fq;
      Msm<Fr, Fq>::g1_to_bytes(ctx->cx, nullptr, points_xy, n, out);
    });
  });
}
int b2m_g1_from_uncompressed(b2m_ctx* ctx, int curve, const uint8_t* bytes, size_t n, uint64_t* out_xy) {
  return guard([&] {
    B2M_REQUIRE(ctx && ((bytes && out_xy) || n == 0), B2M_ERR_INVALID_ARG, "null argument");
    ctx->cx.use();
    with_curve(curve, [&](auto t) {
      using Fr = typename decltype(t)::Fr;
      using Fq = typename decltype(t)::Fq;
      Msm<Fr, Fq>::g1_from_bytes(ctx->cx, bytes, n, out_xy);
    });
  });
}

static int ark_fail(const ArkBad& bad, size_t* bad_index, int* bad_reason) {
  if (bad_index) *bad_index = bad.index;
  if (bad_reason) *bad_reason = bad.reason;
  return bad.reason == G1_OK ? B2M_OK : B2M_ERR_SERIALIZATION;
}
int b2m_g1_decode_ark(b2m_ctx* ctx, int curve, const uint8_t* bytes, size_t n, int compressed, uint64_t* out_xy, size_t* bad_index,
                      int* bad_reason) {
  return guard([&] {
    B2M_REQUIRE(ctx && ((bytes && out_xy) || n == 0), B2M_ERR_INVALID_ARG, "null argument");
    require_curve(curve);
    ctx->cx.use();
    const ArkBad bad = n == 0 ? ArkBad{0, G1_OK} : with_curve(curve, [&](auto t) {
      return g1_decode_ark<typename decltype(t)::Fq>(ctx->cx, bytes, n, compressed != 0, out_xy);
    });
    if (ark_fail(bad, bad_index, bad_reason) != B2M_OK)
      throw Error(B2M_ERR_SERIALIZATION, fmt("G1 point %zu: %s", bad.index, point_status_name(bad.reason)));
  });
}
int b2m_g2_decode_ark(b2m_ctx* ctx, int curve, const uint8_t* bytes, size_t n, int compressed, uint8_t* out_uncompressed, size_t* bad_index,
                      int* bad_reason) {
  return guard([&] {
    B2M_REQUIRE(ctx && ((bytes && out_uncompressed) || n == 0), B2M_ERR_INVALID_ARG, "null argument");
    require_curve(curve);
    ctx->cx.use();
    const ArkBad bad = n == 0 ? ArkBad{0, G1_OK} : with_curve(curve, [&](auto t) {
      return g2_decode_ark<typename decltype(t)::Fq>(ctx->cx, bytes, n, compressed != 0, out_uncompressed);
    });
    if (ark_fail(bad, bad_index, bad_reason) != B2M_OK)
      throw Error(B2M_ERR_SERIALIZATION, fmt("G2 point %zu: %s", bad.index, point_status_name(bad.reason)));
  });
}
int b2m_g1_decode_lem(b2m_ctx* ctx, int curve, const uint8_t* bytes, size_t n, uint64_t* out_xy, size_t* bad_index, int* bad_reason) {
  return guard([&] {
    B2M_REQUIRE(ctx && ((bytes && out_xy) || n == 0), B2M_ERR_INVALID_ARG, "null argument");
    require_curve(curve);
    ctx->cx.use();
    const ArkBad bad = n == 0 ? ArkBad{0, G1_OK} : with_curve(curve, [&](auto t) {
      return g1_decode_lem_points<typename decltype(t)::Fq>(ctx->cx, bytes, n, out_xy);
    });
    if (ark_fail(bad, bad_index, bad_reason) != B2M_OK)
      throw Error(B2M_ERR_SERIALIZATION, fmt("G1 point %zu: %s", bad.index, point_status_name(bad.reason)));
  });
}
int b2m_g2_decode_lem(b2m_ctx* ctx, int curve, const uint8_t* bytes, size_t n, uint8_t* out_uncompressed, size_t* bad_index, int* bad_reason) {
  return guard([&] {
    B2M_REQUIRE(ctx && ((bytes && out_uncompressed) || n == 0), B2M_ERR_INVALID_ARG, "null argument");
    require_curve(curve);
    ctx->cx.use();
    const ArkBad bad = n == 0 ? ArkBad{0, G1_OK} : with_curve(curve, [&](auto t) {
      return g2_decode_lem_points<typename decltype(t)::Fq>(ctx->cx, bytes, n, out_uncompressed);
    });
    if (ark_fail(bad, bad_index, bad_reason) != B2M_OK)
      throw Error(B2M_ERR_SERIALIZATION, fmt("G2 point %zu: %s", bad.index, point_status_name(bad.reason)));
  });
}
int b2m_pairing_check(b2m_ctx* ctx, int curve, size_t n_g2, const uint8_t* g2, size_t n_products, const size_t* product_off,
                      const uint64_t* g1_xy, const uint32_t* g2_index, int* verdicts) {
  return guard([&] {
    B2M_REQUIRE(ctx && (g2 || n_g2 == 0) && ((product_off && verdicts) || n_products == 0), B2M_ERR_INVALID_ARG, "null argument");
    B2M_REQUIRE(n_products == 0 || product_off[n_products] == product_off[0] || (g1_xy && g2_index), B2M_ERR_INVALID_ARG, "null argument");
    require_curve(curve);
    ctx->cx.use();
    with_curve(curve, [&](auto t) { pairing_check<typename decltype(t)::Fq>(ctx->cx, n_g2, g2, n_products, product_off, g1_xy, g2_index, verdicts); });
  });
}
int b2m_g1_to_compressed(b2m_ctx* ctx, int curve, const uint64_t* points_xy, size_t n, uint8_t* out) {
  return guard([&] {
    B2M_REQUIRE(ctx && ((points_xy && out) || n == 0), B2M_ERR_INVALID_ARG, "null argument");
    ctx->cx.use();
    if (n == 0) return;
    with_curve(curve, [&](auto t) { g1_to_compressed<typename decltype(t)::Fq>(ctx->cx, points_xy, n, out); });
  });
}
int b2m_g2_to_compressed(int curve, const uint8_t* uncompressed, size_t n, uint8_t* out) {
  return guard([&] {
    B2M_REQUIRE((uncompressed && out) || n == 0, B2M_ERR_INVALID_ARG, "null argument");
    with_curve(curve, [&](auto t) {
      using Fq = typename decltype(t)::Fq;
      for (size_t i = 0; i < n; i++) g2_compress<Fq>(uncompressed + i * 4 * Fq::N * 4, out + i * 2 * Fq::N * 4);
    });
  });
}

}  // extern "C"
template <class Fr>
static void fr_decode_host(Ctx& cx, const uint8_t* bytes, size_t n, uint64_t* out, size_t* bad_index) {
  DBuf<Fr> d(cx, n);
  const ArkBad bad = fr_decode_ark<Fr>(cx, bytes, n, d.p);
  if (bad_index) *bad_index = bad.index;
  if (bad.index != n) throw Error(B2M_ERR_SERIALIZATION, fmt("Fr element %zu: not below the field modulus", bad.index));
  d.download(reinterpret_cast<Fr*>(out), n);
  cx.sync();
}
template <class Fr>
static void fr_encode_host(Ctx& cx, const uint64_t* limbs, size_t n, uint8_t* out) {
  DBuf<Fr> d(cx, n);
  d.upload(reinterpret_cast<const Fr*>(limbs), n);
  fr_to_canonical<Fr>(cx, d.p, n, out);
  cx.sync();
}
extern "C" {
int b2m_fr_decode_ark(b2m_ctx* ctx, int curve, const uint8_t* bytes, size_t n, uint64_t* out_limbs, size_t* bad_index) {
  return guard([&] {
    B2M_REQUIRE(ctx && ((bytes && out_limbs) || n == 0), B2M_ERR_INVALID_ARG, "null argument");
    require_curve(curve);
    if (bad_index) *bad_index = n;
    if (n == 0) return;
    ctx->cx.use();
    with_curve(curve, [&](auto t) { fr_decode_host<typename decltype(t)::Fr>(ctx->cx, bytes, n, out_limbs, bad_index); });
  });
}
int b2m_fr_to_canonical(b2m_ctx* ctx, int curve, const uint64_t* limbs, size_t n, uint8_t* out) {
  return guard([&] {
    B2M_REQUIRE(ctx && ((limbs && out) || n == 0), B2M_ERR_INVALID_ARG, "null argument");
    require_curve(curve);
    if (n == 0) return;
    ctx->cx.use();
    with_curve(curve, [&](auto t) { fr_encode_host<typename decltype(t)::Fr>(ctx->cx, limbs, n, out); });
  });
}

// The row-length chain of an ark-serialize `Vec<Vec<T>>` (host; one step per row, nothing else can be done in parallel)
int b2m_ark_matrix_rows(const uint8_t* bytes, size_t len, size_t n_rows, size_t entry_bytes, uint64_t* row_ptr, size_t* end,
                        size_t* bad_row, int* bad_reason) {
  if (end) *end = 0;
  if (bad_row) *bad_row = 0;
  if (bad_reason) *bad_reason = 0;
  return guard([&] {
    B2M_REQUIRE(row_ptr && end && (bytes || len == 0) && entry_bytes >= 1, B2M_ERR_INVALID_ARG, "null argument");
    size_t pos = 0;
    row_ptr[0] = 0;
    for (size_t r = 0; r < n_rows; r++) {
      uint64_t n = 0;
      if (len - pos < 8) {
        *end = pos;
        if (bad_row) *bad_row = r;
        if (bad_reason) *bad_reason = 1;
        throw Error(B2M_ERR_SERIALIZATION, fmt("row %zu: truncated in the row length", r));
      }
      memcpy(&n, bytes + pos, 8);
      if (n > (len - pos - 8) / entry_bytes) {
        *end = pos;
        if (bad_row) *bad_row = r;
        if (bad_reason) *bad_reason = 2;
        throw Error(B2M_ERR_SERIALIZATION, fmt("row %zu: %llu entries run past the end", r, (unsigned long long)n));
      }
      row_ptr[r + 1] = row_ptr[r] + n;
      pos += 8 + n * entry_bytes;
    }
    *end = pos;
  });
}

// The term-count chain of a circom `.r1cs` constraint section (host; one step per linear combination, nothing else can be
// done in parallel).  Entries are (u32 wire, 32-byte coefficient): n8 = 32.
int b2m_circom_constraint_rows(const uint8_t* bytes, size_t len, size_t m, uint64_t* row_ptr_a, uint64_t* row_ptr_b, uint64_t* row_ptr_c,
                               size_t* end, size_t* bad_constraint, int* bad_reason) {
  if (end) *end = 0;
  if (bad_constraint) *bad_constraint = 0;
  if (bad_reason) *bad_reason = 0;
  return guard([&] {
    B2M_REQUIRE(row_ptr_a && row_ptr_b && row_ptr_c && end && (bytes || len == 0), B2M_ERR_INVALID_ARG, "null argument");
    uint64_t* rp[3] = {row_ptr_a, row_ptr_b, row_ptr_c};
    size_t pos = 0;
    for (int j = 0; j < 3; j++) rp[j][0] = 0;
    for (size_t k = 0; k < m; k++) {
      for (int j = 0; j < 3; j++) {
        auto fail = [&](int reason, const std::string& what) {
          *end = pos;
          if (bad_constraint) *bad_constraint = k;
          if (bad_reason) *bad_reason = reason;
          throw Error(B2M_ERR_SERIALIZATION, fmt("constraints[%zu].%c: %s", k, "ABC"[j], what.c_str()));
        };
        if (len - pos < 4) fail(1, "truncated in the term count");
        uint32_t n = 0;
        memcpy(&n, bytes + pos, 4);
        if (n > (len - pos - 4) / CIRCOM_TERM_BYTES) fail(2, fmt("%u terms run past the end of the section", n));
        rp[j][k + 1] = rp[j][k] + n;
        pos += 4 + (size_t)n * CIRCOM_TERM_BYTES;
      }
    }
    *end = pos;
  });
}
int b2m_circom_decode_constraints(b2m_ctx* ctx, int curve, const uint8_t* bytes, size_t len, size_t m, const uint64_t* const* row_ptrs,
                                  uint64_t n_wires, uint64_t ni0, uint64_t shift, uint64_t* const* out_row_ptr, uint64_t* const* out_col,
                                  uint64_t* const* out_coeff, int* bad_matrix, size_t* bad_term, int* bad_reason) {
  if (bad_matrix) *bad_matrix = 0;
  if (bad_term) *bad_term = 0;
  if (bad_reason) *bad_reason = 0;
  return guard([&] {
    B2M_REQUIRE(ctx && row_ptrs && out_row_ptr && out_col && out_coeff && (bytes || len == 0), B2M_ERR_INVALID_ARG, "null argument");
    for (int j = 0; j < 3; j++)
      B2M_REQUIRE(row_ptrs[j] && out_row_ptr[j] && ((out_col[j] && out_coeff[j]) || row_ptrs[j][m] == 0), B2M_ERR_INVALID_ARG, "null argument");
    require_curve(curve);
    ctx->cx.use();
    const CircomBad bad = with_curve(curve, [&](auto t) {
      return circom_decode_constraints<typename decltype(t)::Fr>(ctx->cx, bytes, len, m, row_ptrs, n_wires, ni0, shift, out_row_ptr, out_col, out_coeff);
    });
    if (bad.reason) {
      if (bad_matrix) *bad_matrix = bad.matrix;
      if (bad_term) *bad_term = bad.term;
      if (bad_reason) *bad_reason = bad.reason;
      throw Error(B2M_ERR_SERIALIZATION, fmt("matrix %c term %zu: %s", "ABC"[bad.matrix], bad.term,
                                             bad.reason == 1 ? "wire >= nWires" : "coefficient not below r"));
    }
  });
}
int b2m_r1cs_check(b2m_ctx* ctx, int curve, size_t nc, size_t nv, size_t ni, const b2m_matrix* a, const b2m_matrix* b, const b2m_matrix* c,
                   const uint64_t* instance, const uint64_t* witness, size_t* bad_row) {
  return guard([&] {
    B2M_REQUIRE(ctx && a && b && c && instance && bad_row && (witness || nv == ni), B2M_ERR_INVALID_ARG, "null argument");
    require_curve(curve);
    ctx->cx.use();
    const b2m_matrix* mats[3] = {a, b, c};
    *bad_row = with_curve(curve, [&](auto t) { return r1cs_check<typename decltype(t)::Fr>(ctx->cx, nc, nv, ni, mats, instance, witness); });
  });
}

}  // extern "C"
// `Radix2EvaluationDomain::new(2^log_size)` as ark-serialize writes it [U ark-poly 0.3 domain/radix2]
template <class Fr>
static void domain_ark_impl(unsigned log_size, uint8_t* out) {
  B2M_REQUIRE((int)log_size <= Fr::Params::TWO_ADICITY, B2M_ERR_DEGREE_TOO_LARGE, "2^%u exceeds the 2-adicity of the field", log_size);
  const uint64_t size = (uint64_t)1 << log_size;
  const uint32_t lg = log_size;
  memcpy(out, &size, 8);
  memcpy(out + 8, &lg, 4);
  Fr gen;
  for (int i = 0; i < Fr::N; i++) gen.l[i] = Fr::Params::gen(i);
  const Fr size_f = Fr::from_u64(size), w = Ntt<Fr>::root_of_unity((int)log_size);
  const Fr vals[5] = {size_f, size_f.inverse(), w, w.inverse(), gen.inverse()};
  for (int k = 0; k < 5; k++) {
    const Fr c = vals[k].to_canonical();
    memcpy(out + 12 + k * sizeof(Fr), c.l, sizeof(Fr));
  }
}
extern "C" {
int b2m_domain_ark(int curve, unsigned log_size, uint8_t* out) {
  return guard([&] {
    B2M_REQUIRE(out != nullptr, B2M_ERR_INVALID_ARG, "null argument");
    with_curve(curve, [&](auto t) { domain_ark_impl<typename decltype(t)::Fr>(log_size, out); });
  });
}

}  // extern "C"
// standard G2 generators (canonical x.c0, x.c1, y.c0, y.c1; big-endian hex), checked on-curve / order r in tests/test_srs_files.py
static const char* const G2_GEN_BLS[4] = {
    "024aa2b2f08f0a91260805272dc51051c6e47ad4fa403b02b4510b647ae3d1770bac0326a805bbefd48056c8c121bdb8",
    "13e02b6052719f607dacd3a088274f65596bd0d09920b61ab5da61bbdc7f5049334cf11213945d57e5ac7d055d042b7e",
    "0ce5d527727d6e118cc9cdc6da2e351aadfd9baa8cbdd3a76d429a695160d12c923ac9cc3baca289e193548608b82801",
    "0606c4a02ea734cc32acd2b02bc28b99cb3e287e85a763af267492ab572e99ab3f370d275cec1da1aaa9075ff05f79be"};
static const char* const G2_GEN_BN[4] = {
    "1800deef121f1e76426a00665e5c4479674322d4f75edadd46debd5cd992f6ed", "198e9393920d483a7260bfb731fb5d25f1aa493335a9e71297e485b7aef312c2",
    "12c85ea5db8c6deb4aab71808dcb408fe3d1e7690c43d37b4ce6cc0166fa7daa", "090689d0585ff075ec9e99ad690c3395bc4b313370b38ef355acdadcd122975b"};
static const char* const G2_GEN_BLS377[4] = {  // ark-bls12-377's G2 generator
    "018480be71c785fec89630a2a3841d01c565f071203e50317ea501f557db6b9b71889f52bb53540274e3e48f7c005196",
    "00ea6040e700403170dc5a51b1b140d5532777ee6651cecbe7223ece0799c9de5cf89984bff76fe6b26bfefa6ea16afe",
    "00690d665d446f7bd960736bcbb2efb4de03ed7274b49a58e458c282f832d204f2cf88886d8c7c2ef094094409fd4ddf",
    "00f8169fd28355189e549da3151a70aa61ef11ac3d591bf12463b01acee304c24279b83f5e52270bd9a1cdd185eb8f93"};
template <class Fq>
static const char* const* g2_generator_hex() {
  if constexpr (std::is_same<Fq, FqBls>::value) return G2_GEN_BLS;
  else if constexpr (std::is_same<Fq, FqBn>::value) return G2_GEN_BN;
  else return G2_GEN_BLS377;
}

template <class Fq>
static Fq fq_from_hex(const char* hex) {
  Fq c = Fq::zero();
  const size_t len = strlen(hex);
  for (size_t i = 0; i < len; i++) {
    const char ch = hex[len - 1 - i];
    const uint32_t v = ch >= 'a' ? ch - 'a' + 10 : ch - '0';
    c.l[i / 8] |= v << (4 * (i % 8));
  }
  return Fq::from_canonical(c);
}
template <class Fq>
static void g2_scalar_muls_impl(const char* const gen[4], const uint8_t* h_bytes, const uint64_t* scalars, size_t n, uint8_t* out) {
  G2Jac<Fq> h;
  if (h_bytes) {
    Fq parts[4];
    for (int k = 0; k < 4; k++) {
      Fq c;
      memcpy(c.l, h_bytes + (size_t)k * Fq::N * 4, Fq::N * 4);
      if (k == 3) {
        B2M_REQUIRE(!((c.l[Fq::N - 1] >> 30) & 1u), B2M_ERR_INVALID_ARG, "the G2 base is the point at infinity");
        c.l[Fq::N - 1] &= 0x3fffffffu;
      }
      parts[k] = Fq::from_canonical(c);
    }
    h = G2Jac<Fq>{Fq2<Fq>{parts[0], parts[1]}, Fq2<Fq>{parts[2], parts[3]}, Fq2<Fq>::one()};
  } else {
    h = G2Jac<Fq>{Fq2<Fq>{fq_from_hex<Fq>(gen[0]), fq_from_hex<Fq>(gen[1])}, Fq2<Fq>{fq_from_hex<Fq>(gen[2]), fq_from_hex<Fq>(gen[3])}, Fq2<Fq>::one()};
  }
  std::vector<uint8_t> bytes;
  for (size_t i = 0; i < n; i++) g2_write_uncompressed<Fq>(bytes, h.mul(reinterpret_cast<const uint32_t*>(scalars + 4 * i), 8));
  memcpy(out, bytes.data(), bytes.size());
}
extern "C" {
int b2m_g2_scalar_muls(int curve, const uint8_t* h_uncompressed, const uint64_t* scalars, size_t n, uint8_t* out) {
  return guard([&] {
    B2M_REQUIRE((scalars && out) || n == 0, B2M_ERR_INVALID_ARG, "null argument");
    with_curve(curve, [&](auto t) {
      using Fq = typename decltype(t)::Fq;
      g2_scalar_muls_impl<Fq>(g2_generator_hex<Fq>(), h_uncompressed, scalars, n, out);
    });
  });
}

// ---- Level 1 ----------------------------------------------------------------------------------
}  // extern "C"
static decltype(&pc_open_combinations_bls) pc_open_combinations_of(int curve) {
  return curve == B2M_CURVE_BLS12_381 ? pc_open_combinations_bls : curve == B2M_CURVE_BN254 ? pc_open_combinations_bn : pc_open_combinations_bls377;
}
extern "C" {
int b2m_pc_commit(b2m_srs* srs, int pc_variant, size_t n_polys, const uint64_t* const* coeffs, const size_t* n_coeffs,
                  const int64_t* degree_bounds, const int64_t* hiding_bounds, b2m_rng* rng, uint64_t* out_comm_xy,
                  uint64_t* out_shifted_xy, uint64_t* out_rand, uint64_t* out_shifted_rand, size_t rand_stride) {
  return guard([&] {
    B2M_REQUIRE(srs && coeffs && n_coeffs && degree_bounds && hiding_bounds && out_comm_xy && out_rand, B2M_ERR_INVALID_ARG, "null argument");
    B2M_REQUIRE(pc_variant == B2M_PC_MARLIN_KZG10 || pc_variant == B2M_PC_SONIC_KZG10, B2M_ERR_INVALID_ARG, "unknown PC variant");
    B2M_REQUIRE(pc_variant != B2M_PC_MARLIN_KZG10 || (out_shifted_xy && out_shifted_rand), B2M_ERR_INVALID_ARG,
                "MarlinKZG10 needs the shifted output buffers");
    B2M_REQUIRE(rng == nullptr || rng->kind == B2M_RNG_CHACHA8 || rng->kind == B2M_RNG_CHACHA12 || rng->kind == B2M_RNG_CHACHA20 ||
                    (rng->kind == B2M_RNG_CALLBACK && rng->next_u64 != nullptr),
                B2M_ERR_MISSING_RNG, "unsupported rng kind");
    srs->ctx->cx.use();
    const auto commit = srs->curve == B2M_CURVE_BLS12_381 ? pc_commit_bls : srs->curve == B2M_CURVE_BN254 ? pc_commit_bn : pc_commit_bls377;
    commit(srs, pc_variant, n_polys, coeffs, n_coeffs, degree_bounds, hiding_bounds, rng, out_comm_xy, out_shifted_xy, out_rand, out_shifted_rand,
           rand_stride);
  });
}

int b2m_pc_open(b2m_srs* srs, int pc_variant, size_t n_polys, const uint64_t* const* coeffs, const size_t* n_coeffs,
                const int64_t* degree_bounds, const uint64_t* rands, const uint64_t* shifted_rands, size_t rand_stride,
                int64_t max_degree_bound, const uint64_t* point, const uint64_t* opening_challenge, uint64_t* out_w_xy,
                int* out_has_random_v, uint64_t* out_random_v) {
  return guard([&] {
    B2M_REQUIRE(srs && coeffs && n_coeffs && degree_bounds && point && opening_challenge && out_w_xy && out_has_random_v && out_random_v,
                B2M_ERR_INVALID_ARG, "null argument");
    B2M_REQUIRE(pc_variant == B2M_PC_MARLIN_KZG10 || pc_variant == B2M_PC_SONIC_KZG10, B2M_ERR_INVALID_ARG, "unknown PC variant");
    B2M_REQUIRE(n_polys >= 1, B2M_ERR_INVALID_ARG, "no polynomials");
    srs->ctx->cx.use();
    // open_combinations with one coefficient-one combination per polynomial, all queried at the one point; null rands
    // give empty randomness
    std::vector<int> hiding(n_polys, 1);
    std::vector<size_t> term_off(n_polys + 1), lc(n_polys), at_point(n_polys, 0);
    std::vector<int64_t> poly(n_polys);
    std::vector<uint64_t> ones(4 * n_polys);
    for (size_t i = 0; i < n_polys; i++) {
      term_off[i + 1] = i + 1;
      lc[i] = i;
      poly[i] = (int64_t)i;
      with_curve(srs->curve, [&](auto t) { memcpy(&ones[4 * i], decltype(t)::Fr::one().l, 32); });
    }
    pc_open_combinations_of(srs->curve)(srs, pc_variant, max_degree_bound, n_polys, coeffs, n_coeffs, degree_bounds, hiding.data(), rands,
                                        shifted_rands, rand_stride, n_polys, term_off.data(), poly.data(), ones.data(), n_polys, lc.data(),
                                        at_point.data(), 1, point, opening_challenge, out_w_xy, out_has_random_v, out_random_v);
  });
}

int b2m_trim(b2m_srs* srs, int pc_variant, size_t supported_degree, size_t supported_hiding_bound, const uint64_t* enforced_degree_bounds,
             size_t n_bounds, b2m_ck** out) {
  return guard([&] {
    B2M_REQUIRE(srs && out && (enforced_degree_bounds || n_bounds == 0), B2M_ERR_INVALID_ARG, "null argument");
    B2M_REQUIRE(pc_variant == B2M_PC_MARLIN_KZG10 || pc_variant == B2M_PC_SONIC_KZG10, B2M_ERR_INVALID_ARG, "unknown PC variant");
    const size_t D = srs->n_g - 1;
    B2M_REQUIRE(supported_degree >= 1 && supported_degree <= D, B2M_ERR_DEGREE_TOO_LARGE, "supported degree %zu out of range (max degree %zu)",
                supported_degree, D);  // TrimmingDegreeTooLarge / DegreeIsZero
    std::unique_ptr<b2m_ck> ck(new b2m_ck{srs, pc_variant, supported_degree, supported_hiding_bound, {}});
    for (size_t k = 0; k < n_bounds; k++) {
      B2M_REQUIRE(enforced_degree_bounds[k] <= supported_degree, B2M_ERR_DEGREE_TOO_LARGE, "enforced degree bound %llu exceeds the supported degree %zu",
                  (unsigned long long)enforced_degree_bounds[k], supported_degree);
      ck->bounds.push_back(enforced_degree_bounds[k]);
    }
    std::sort(ck->bounds.begin(), ck->bounds.end());
    ck->bounds.erase(std::unique(ck->bounds.begin(), ck->bounds.end()), ck->bounds.end());
    // the hiding powers this key will be asked for must be resident (throws B2M_ERR_INVALID_ARG naming the missing power)
    for (size_t i = 0; i <= supported_hiding_bound + 1; i++) srs->gamma_slot(i);
    if (pc_variant == B2M_PC_SONIC_KZG10)
      for (uint64_t b : ck->bounds)
        for (size_t i = 0; i <= supported_hiding_bound + 1; i++) srs->gamma_slot(D - b + i);
    *out = ck.release();
    srs->children++;
  });
}

void b2m_ck_destroy(b2m_ck* ck) {
  if (!ck) return;
  b2m_srs* srs = ck->srs;
  delete ck;
  if (--srs->children == 0 && srs->dead) b2m_release_srs(srs);
}

size_t b2m_ck_supported_degree(const b2m_ck* ck) { return ck ? ck->supported_degree : 0; }

int b2m_ck_shift_power(const b2m_ck* ck, uint64_t bound, uint64_t* out_xy) {
  return guard([&] {
    B2M_REQUIRE(ck && out_xy, B2M_ERR_INVALID_ARG, "null argument");
    B2M_REQUIRE(ck->enforced(bound), B2M_ERR_INVALID_ARG, "degree bound %llu is not enforced by this committer key", (unsigned long long)bound);
    b2m_srs* srs = ck->srs;
    srs->ctx->cx.use();
    const size_t slot = srs->n_g - 1 - bound;
    with_curve(srs->curve, [&](auto t) { srs->msm<typename decltype(t)::Fr>()->read_power(slot, out_xy); });
  });
}

static void ck_check_polys(const b2m_ck* ck, size_t n_polys, const size_t* n_coeffs, const int64_t* degree_bounds, const int64_t* hiding_bounds) {
  for (size_t i = 0; i < n_polys; i++) {
    B2M_REQUIRE(n_coeffs[i] <= ck->supported_degree + 1, B2M_ERR_DEGREE_TOO_LARGE, "polynomial %zu has degree %zu, the committer key supports %zu", i,
                n_coeffs[i] ? n_coeffs[i] - 1 : 0, ck->supported_degree);  // TooManyCoefficients
    if (degree_bounds[i] >= 0)
      B2M_REQUIRE(ck->enforced((uint64_t)degree_bounds[i]), B2M_ERR_INVALID_ARG, "polynomial %zu: degree bound %lld is not enforced by this committer key", i,
                  (long long)degree_bounds[i]);  // UnsupportedDegreeBound
    if (hiding_bounds && hiding_bounds[i] >= 0)
      B2M_REQUIRE((size_t)hiding_bounds[i] <= ck->hiding_bound, B2M_ERR_INVALID_ARG, "polynomial %zu: hiding bound %lld above the supported %zu", i,
                  (long long)hiding_bounds[i], ck->hiding_bound);  // HidingBoundToolarge
  }
}

int b2m_ck_commit(b2m_ck* ck, size_t n_polys, const uint64_t* const* coeffs, const size_t* n_coeffs, const int64_t* degree_bounds,
                  const int64_t* hiding_bounds, b2m_rng* rng, uint64_t* out_comm_xy, uint64_t* out_shifted_xy, uint64_t* out_rand,
                  uint64_t* out_shifted_rand, size_t rand_stride) {
  int rc = guard([&] {
    B2M_REQUIRE(ck && n_coeffs && degree_bounds && hiding_bounds, B2M_ERR_INVALID_ARG, "null argument");
    ck_check_polys(ck, n_polys, n_coeffs, degree_bounds, hiding_bounds);
  });
  if (rc != B2M_OK) return rc;
  return b2m_pc_commit(ck->srs, ck->pc, n_polys, coeffs, n_coeffs, degree_bounds, hiding_bounds, rng, out_comm_xy, out_shifted_xy, out_rand,
                       out_shifted_rand, rand_stride);
}

int b2m_ck_open_combinations(b2m_ck* ck, size_t n_polys, const uint64_t* const* coeffs, const size_t* n_coeffs, const int64_t* degree_bounds,
                             const int* hiding, const uint64_t* rands, const uint64_t* shifted_rands, size_t rand_stride, size_t n_lcs,
                             const size_t* lc_term_off, const int64_t* lc_poly, const uint64_t* lc_coeff, size_t n_queries, const size_t* query_lc,
                             const size_t* query_point, size_t n_points, const uint64_t* points, const uint64_t* opening_challenge,
                             uint64_t* out_w_xy, int* out_has_random_v, uint64_t* out_random_v) {
  return guard([&] {
    B2M_REQUIRE(ck && coeffs && n_coeffs && degree_bounds && hiding && rands && lc_term_off && lc_poly && lc_coeff && query_lc && query_point &&
                    points && opening_challenge && out_w_xy && out_has_random_v && out_random_v,
                B2M_ERR_INVALID_ARG, "null argument");
    B2M_REQUIRE(n_polys >= 1 && n_lcs >= 1 && n_points >= 1 && n_queries >= 1, B2M_ERR_INVALID_ARG, "empty opening");
    B2M_REQUIRE(ck->pc != B2M_PC_MARLIN_KZG10 || shifted_rands, B2M_ERR_INVALID_ARG, "MarlinKZG10 needs the shifted randomness");
    ck_check_polys(ck, n_polys, n_coeffs, degree_bounds, nullptr);
    for (size_t q = 0; q < n_queries; q++) B2M_REQUIRE(query_point[q] < n_points, B2M_ERR_INVALID_ARG, "query %zu names point %zu of %zu", q, query_point[q], n_points);
    b2m_srs* srs = ck->srs;
    srs->ctx->cx.use();
    pc_open_combinations_of(srs->curve)(srs, ck->pc, ck->max_bound(), n_polys, coeffs, n_coeffs, degree_bounds, hiding, rands, shifted_rands,
                                        rand_stride, n_lcs, lc_term_off, lc_poly, lc_coeff, n_queries, query_lc, query_point, n_points, points,
                                        opening_challenge, out_w_xy, out_has_random_v, out_random_v);
  });
}

// ---- Level 2 ----------------------------------------------------------------------------------
struct b2m_index {
  b2m_srs* srs;
  std::unique_ptr<IndexBase> impl;
};

int b2m_index_create(b2m_srs* srs, int pc_variant, size_t num_constraints, size_t num_variables, size_t num_instance_variables,
                     const b2m_matrix* a, const b2m_matrix* b, const b2m_matrix* c, b2m_index** out) {
  return guard([&] {
    B2M_REQUIRE(srs && a && b && c && out, B2M_ERR_INVALID_ARG, "null argument");
    B2M_REQUIRE(pc_variant == B2M_PC_MARLIN_KZG10 || pc_variant == B2M_PC_SONIC_KZG10, B2M_ERR_INVALID_ARG, "unknown PC variant");
    srs->ctx->cx.use();
    std::unique_ptr<b2m_index> idx(new b2m_index);
    idx->srs = srs;
    const auto make = srs->curve == B2M_CURVE_BLS12_381 ? make_index_bls : srs->curve == B2M_CURVE_BN254 ? make_index_bn : make_index_bls377;
    idx->impl.reset(make(srs, pc_variant, num_constraints, num_variables, num_instance_variables, a, b, c));
    *out = idx.release();
    srs->children++;
  });
}

int b2m_index_load(b2m_srs* srs, int pc_variant, size_t num_constraints, size_t num_variables, size_t num_instance_variables,
                   size_t num_non_zero, const b2m_matrix* a, const b2m_matrix* b, const b2m_matrix* c, const uint8_t* const* vectors,
                   const size_t* vector_lens, const uint64_t* index_comms_xy, int check_commitments, size_t* bad_vector, size_t* bad_index,
                   int* bad_reason, b2m_index** out) {
  size_t bad[3] = {0, 0, 0};
  const int rc = guard([&] {
    B2M_REQUIRE(srs && a && b && c && vectors && vector_lens && index_comms_xy && out, B2M_ERR_INVALID_ARG, "null argument");
    B2M_REQUIRE(pc_variant == B2M_PC_MARLIN_KZG10 || pc_variant == B2M_PC_SONIC_KZG10, B2M_ERR_INVALID_ARG, "unknown PC variant");
    for (int v = 0; v < 12; v++) B2M_REQUIRE(vectors[v] || vector_lens[v] == 0, B2M_ERR_INVALID_ARG, "index vector %d is null", v);
    srs->ctx->cx.use();
    std::unique_ptr<b2m_index> idx(new b2m_index);
    idx->srs = srs;
    const auto load = srs->curve == B2M_CURVE_BLS12_381 ? load_index_bls : srs->curve == B2M_CURVE_BN254 ? load_index_bn : load_index_bls377;
    idx->impl.reset(load(srs, pc_variant, num_constraints, num_variables, num_instance_variables, num_non_zero, a, b, c, vectors, vector_lens,
                         index_comms_xy, check_commitments != 0, bad));
    *out = idx.release();
    srs->children++;
  });
  if (bad_vector) *bad_vector = bad[0];
  if (bad_index) *bad_index = bad[1];
  if (bad_reason) *bad_reason = rc == B2M_ERR_SERIALIZATION ? (int)bad[2] : 0;
  return rc;
}

int b2m_index_sizes(const b2m_index* idx, size_t* num_non_zero, size_t* domain_k, size_t* matrix_nnz) {
  return guard([&] {
    B2M_REQUIRE(idx && num_non_zero && domain_k && matrix_nnz, B2M_ERR_INVALID_ARG, "null argument");
    idx->impl->sizes(num_non_zero, domain_k, matrix_nnz);
  });
}

int b2m_index_export(b2m_index* idx, uint8_t* vectors, uint64_t* const* row_ptrs, uint64_t* const* cols, uint8_t* const* coeffs) {
  return guard([&] {
    B2M_REQUIRE(idx != nullptr, B2M_ERR_INVALID_ARG, "null argument");
    idx->srs->ctx->cx.use();
    idx->impl->export_keys(vectors, row_ptrs, cols, coeffs);
  });
}

int b2m_index_residency(const b2m_index* idx, int* host, size_t* host_bytes) {
  return guard([&] {
    B2M_REQUIRE(idx != nullptr, B2M_ERR_INVALID_ARG, "null argument");
    if (host) *host = idx->impl->host_resident;
    if (host_bytes) *host_bytes = idx->impl->host_bytes;
  });
}

void b2m_index_destroy(b2m_index* idx) {
  if (!idx) return;
  b2m_srs* srs = idx->srs;
  srs->ctx->cx.use();
  cudaStreamSynchronize(srs->ctx->cx.stream);
  delete idx;
  if (--srs->children == 0 && srs->dead) b2m_release_srs(srs);
}

int b2m_index_vk_bytes(const b2m_index* idx, uint8_t* out, size_t cap, size_t* len) {
  return guard([&] {
    B2M_REQUIRE(idx && len, B2M_ERR_INVALID_ARG, "null argument");
    *len = idx->impl->vk_bytes.size();
    if (out) {
      B2M_REQUIRE(cap >= *len, B2M_ERR_INVALID_ARG, "buffer too small (%zu < %zu)", cap, *len);
      memcpy(out, idx->impl->vk_bytes.data(), *len);
    }
  });
}

int b2m_index_comms(const b2m_index* idx, uint64_t* out_xy) {
  return guard([&] {
    B2M_REQUIRE(idx && out_xy, B2M_ERR_INVALID_ARG, "null argument");
    memcpy(out_xy, idx->impl->comms_xy.data(), idx->impl->comms_xy.size() * sizeof(uint64_t));
  });
}

int b2m_prove(b2m_index* idx, const uint64_t* formatted_input, size_t n_input, const uint64_t* witness, size_t n_witness,
              b2m_rng* zk_rng, uint8_t* proof, size_t cap, size_t* proof_len) {
  return guard([&] {
    B2M_REQUIRE(idx && proof && proof_len, B2M_ERR_INVALID_ARG, "null argument");
    B2M_REQUIRE(formatted_input == nullptr || witness || n_witness == 0, B2M_ERR_INVALID_ARG, "null witness");
    B2M_REQUIRE(zk_rng != nullptr, B2M_ERR_MISSING_RNG, "zk_rng is required (hiding commitments)");
    idx->srs->ctx->cx.use();
    std::vector<uint8_t> bytes;
    idx->impl->prove(formatted_input, n_input, witness, n_witness, zk_rng, bytes);
    *proof_len = bytes.size();
    B2M_REQUIRE(cap >= bytes.size(), B2M_ERR_INVALID_ARG, "proof buffer too small (%zu < %zu)", cap, bytes.size());
    memcpy(proof, bytes.data(), bytes.size());
  });
}

int b2m_index_stage(b2m_index* idx, const uint64_t* formatted_input, size_t n_input, const uint64_t* witness, size_t n_witness) {
  return guard([&] {
    B2M_REQUIRE(idx && formatted_input && (witness || n_witness == 0), B2M_ERR_INVALID_ARG, "null argument");
    idx->srs->ctx->cx.use();
    idx->impl->stage(formatted_input, n_input, witness, n_witness);
  });
}

int b2m_prove_timings(const b2m_index* idx, char* json, size_t cap) {
  return guard([&] {
    B2M_REQUIRE(idx && json && cap > 0, B2M_ERR_INVALID_ARG, "null argument");
    snprintf(json, cap, "%s", idx->impl->timings_json.c_str());
  });
}

// ---- Level 2: verifier ----------------------------------------------------------------------------
struct b2m_vk {
  b2m_ctx* ctx;
  int curve;
  std::unique_ptr<VerifierBase> impl;
};

// the batch randomisers must be unpredictable to the prover: a verify call without a usable rng is refused
static void require_verify_rng(const b2m_rng* rng) {
  B2M_REQUIRE(rng != nullptr, B2M_ERR_MISSING_RNG, "rng is required (the batch randomisers must be unpredictable to the prover)");
  B2M_REQUIRE(rng->kind == B2M_RNG_CHACHA8 || rng->kind == B2M_RNG_CHACHA12 || rng->kind == B2M_RNG_CHACHA20 ||
                  (rng->kind == B2M_RNG_CALLBACK && rng->next_u64 != nullptr),
              B2M_ERR_MISSING_RNG, "unsupported rng kind %d", rng->kind);
}

int b2m_vk_create(b2m_ctx* ctx, int curve, int pc_variant, size_t num_constraints, size_t num_variables, size_t num_non_zero,
                  const uint64_t* index_comms_xy, const uint64_t* g_xy, const uint64_t* gamma_g_xy, const uint8_t* h_bytes,
                  const uint8_t* beta_h_bytes, size_t n_bounds, const uint64_t* bounds, const void* bound_points, b2m_vk** out) {
  return guard([&] {
    B2M_REQUIRE(ctx && index_comms_xy && g_xy && gamma_g_xy && h_bytes && beta_h_bytes && out && (n_bounds == 0 || (bounds && bound_points)),
                B2M_ERR_INVALID_ARG, "null argument");
    require_curve(curve);
    B2M_REQUIRE(pc_variant == B2M_PC_MARLIN_KZG10 || pc_variant == B2M_PC_SONIC_KZG10, B2M_ERR_INVALID_ARG, "unknown PC variant");
    B2M_REQUIRE(ctx->cx.world <= 1, B2M_ERR_UNSUPPORTED, "verification on a multi-GPU context");
    ctx->cx.use();
    const VkArgs a{pc_variant, num_constraints, num_variables, num_non_zero, index_comms_xy, g_xy, gamma_g_xy, h_bytes, beta_h_bytes,
                   n_bounds, bounds, bound_points};
    std::unique_ptr<b2m_vk> vk(new b2m_vk{ctx, curve, nullptr});
    const auto make = curve == B2M_CURVE_BLS12_381 ? make_verifier_bls : curve == B2M_CURVE_BN254 ? make_verifier_bn : make_verifier_bls377;
    vk->impl.reset(make(ctx->cx, a));
    *out = vk.release();
    ctx->children++;
  });
}

void b2m_vk_destroy(b2m_vk* vk) {
  if (!vk) return;
  b2m_ctx* ctx = vk->ctx;
  ctx->cx.use();
  cudaStreamSynchronize(ctx->cx.stream);
  delete vk;
  if (--ctx->children == 0 && ctx->dead) b2m_release_ctx(ctx);
}

int b2m_verify_batch(b2m_vk* vk, size_t n, const uint64_t* const* public_inputs, const size_t* n_inputs, const uint8_t* const* proofs,
                     const size_t* proof_lens, b2m_rng* rng, int* verdicts) {
  return guard([&] {
    B2M_REQUIRE(vk && (n == 0 || (public_inputs && n_inputs && proofs && proof_lens && verdicts)), B2M_ERR_INVALID_ARG, "null argument");
    require_verify_rng(rng);
    for (size_t i = 0; i < n; i++) B2M_REQUIRE(public_inputs[i] || n_inputs[i] == 0, B2M_ERR_INVALID_ARG, "public input %zu is null", i);
    vk->ctx->cx.use();
    vk->impl->verify_batch(n, public_inputs, n_inputs, proofs, proof_lens, rng, verdicts);
  });
}

int b2m_verify_multi(size_t n_keys, b2m_vk* const* vks, size_t n, const uint32_t* key_of, const uint64_t* const* public_inputs,
                     const size_t* n_inputs, const uint8_t* const* proofs, const size_t* proof_lens, b2m_rng* rng, int* verdicts) {
  return guard([&] {
    B2M_REQUIRE((n_keys == 0 || vks) && (n == 0 || (key_of && public_inputs && n_inputs && proofs && proof_lens && verdicts)), B2M_ERR_INVALID_ARG,
                "null argument");
    for (size_t k = 0; k < n_keys; k++) {
      B2M_REQUIRE(vks[k], B2M_ERR_INVALID_ARG, "key %zu is null", k);
      B2M_REQUIRE(vks[k]->ctx == vks[0]->ctx, B2M_ERR_INVALID_ARG, "key %zu belongs to another context than key 0", k);
      B2M_REQUIRE(vks[k]->curve == vks[0]->curve, B2M_ERR_INVALID_ARG, "key %zu is on curve %d, key 0 on curve %d", k, vks[k]->curve, vks[0]->curve);
    }
    for (size_t i = 0; i < n; i++) B2M_REQUIRE(key_of[i] < n_keys, B2M_ERR_INVALID_ARG, "key_of[%zu] = %u is not below n_keys = %zu", i, key_of[i], n_keys);
    require_verify_rng(rng);
    for (size_t i = 0; i < n; i++) B2M_REQUIRE(public_inputs[i] || n_inputs[i] == 0, B2M_ERR_INVALID_ARG, "public input %zu is null", i);
    if (n_keys == 0) return;  // (and so n == 0)
    std::vector<VerifierBase*> impls(n_keys);
    for (size_t k = 0; k < n_keys; k++) impls[k] = vks[k]->impl.get();
    vks[0]->ctx->cx.use();
    impls[0]->verify_multi(n_keys, impls.data(), n, key_of, public_inputs, n_inputs, proofs, proof_lens, rng, verdicts);
  });
}

int b2m_srs_check_powers(b2m_srs* srs, const uint8_t* h, const uint8_t* beta_h, size_t n_neg, const uint64_t* neg_keys, const uint8_t* neg_h,
                         b2m_rng* rng, int* ok, int* bad_kind, size_t* bad_index) {
  return guard([&] {
    B2M_REQUIRE(srs && h && beta_h && ok && (n_neg == 0 || (neg_keys && neg_h)), B2M_ERR_INVALID_ARG, "null argument");
    B2M_REQUIRE(srs->ctx->cx.world <= 1, B2M_ERR_UNSUPPORTED, "the power check on a multi-GPU context");
    require_verify_rng(rng);
    *ok = 0;
    srs->ctx->cx.use();
    with_curve(srs->curve, [&](auto t) {
      srs_check_powers<typename decltype(t)::Fr, typename decltype(t)::Fq>(srs, h, beta_h, n_neg, neg_keys, neg_h, rng, ok, bad_kind, bad_index);
    });
  });
}

// ---- Level 1: PC verifier -------------------------------------------------------------------------
struct b2m_pc_vk {
  b2m_ctx* ctx;
  int pc;
  std::unique_ptr<PcVerifierBase> impl;
};

int b2m_pc_vk_create(b2m_ctx* ctx, int curve, int pc_variant, size_t max_degree, const uint64_t* g_xy, const uint64_t* gamma_g_xy,
                     const uint8_t* h_bytes, const uint8_t* beta_h_bytes, size_t n_bounds, const uint64_t* bounds, const void* bound_points,
                     b2m_pc_vk** out) {
  return guard([&] {
    B2M_REQUIRE(ctx && g_xy && gamma_g_xy && h_bytes && beta_h_bytes && out && (n_bounds == 0 || (bounds && bound_points)), B2M_ERR_INVALID_ARG,
                "null argument");
    require_curve(curve);
    B2M_REQUIRE(pc_variant == B2M_PC_MARLIN_KZG10 || pc_variant == B2M_PC_SONIC_KZG10, B2M_ERR_INVALID_ARG, "unknown PC variant");
    B2M_REQUIRE(ctx->cx.world <= 1, B2M_ERR_UNSUPPORTED, "verification on a multi-GPU context");
    ctx->cx.use();
    const PcVkArgs a{pc_variant, max_degree, g_xy, gamma_g_xy, h_bytes, beta_h_bytes, n_bounds, bounds, bound_points};
    std::unique_ptr<b2m_pc_vk> vk(new b2m_pc_vk{ctx, pc_variant, nullptr});
    const auto make = curve == B2M_CURVE_BLS12_381 ? make_pc_verifier_bls : curve == B2M_CURVE_BN254 ? make_pc_verifier_bn : make_pc_verifier_bls377;
    vk->impl.reset(make(ctx->cx, a));
    *out = vk.release();
    ctx->children++;
  });
}

void b2m_pc_vk_destroy(b2m_pc_vk* vk) {
  if (!vk) return;
  b2m_ctx* ctx = vk->ctx;
  ctx->cx.use();
  cudaStreamSynchronize(ctx->cx.stream);
  delete vk;
  if (--ctx->children == 0 && ctx->dead) b2m_release_ctx(ctx);
}

int b2m_pc_check_combinations(b2m_pc_vk* vk, size_t n_sets, const size_t* comm_off, const uint8_t* comms, const int64_t* comm_bounds,
                              const int* has_shifted, const uint8_t* shifted, const size_t* lc_off, const size_t* lc_term_off,
                              const int64_t* lc_comm, const uint64_t* lc_coeff, const size_t* point_off, const uint64_t* points,
                              const uint8_t* w, const int* has_random_v, const uint8_t* random_v, const size_t* query_off,
                              const size_t* query_lc, const size_t* query_point, const uint8_t* evals, const uint64_t* challenges,
                              b2m_rng* rng, int* verdicts) {
  return guard([&] {
    B2M_REQUIRE(vk && (n_sets == 0 || (comm_off && lc_off && lc_term_off && point_off && query_off && challenges && verdicts)), B2M_ERR_INVALID_ARG,
                "null argument");
    const PcSets S{n_sets, comm_off, comms, comm_bounds, has_shifted, shifted, lc_off, lc_term_off, lc_comm, lc_coeff, point_off, points, w,
                   has_random_v, random_v, query_off, query_lc, query_point, evals, challenges};
    if (n_sets) {  // the arrays a non-empty range reads
      const size_t nc = comm_off[n_sets] - comm_off[0], nt = lc_term_off[lc_off[n_sets]] - lc_term_off[lc_off[0]];
      const size_t np = point_off[n_sets] - point_off[0], nq = query_off[n_sets] - query_off[0];
      B2M_REQUIRE((nc == 0 || (comms && comm_bounds && (vk->pc == B2M_PC_SONIC_KZG10 || (has_shifted && shifted)))) && (nt == 0 || (lc_comm && lc_coeff)) &&
                      (np == 0 || (points && w && has_random_v && random_v)) && (nq == 0 || (query_lc && query_point && evals)),
                  B2M_ERR_INVALID_ARG, "null argument");
    }
    require_verify_rng(rng);
    vk->ctx->cx.use();
    vk->impl->check_combinations(S, rng, verdicts);
  });
}

int b2m_pc_vk_timings(const b2m_pc_vk* vk, char* json, size_t cap) {
  return guard([&] {
    B2M_REQUIRE(vk && json && cap > 0, B2M_ERR_INVALID_ARG, "null argument");
    snprintf(json, cap, "%s", vk->impl->timings_json.c_str());
  });
}

int b2m_verify(b2m_vk* vk, const uint64_t* public_input, size_t n_input, const uint8_t* proof, size_t proof_len, b2m_rng* rng, int* ok) {
  int rc = guard([&] { B2M_REQUIRE(ok != nullptr, B2M_ERR_INVALID_ARG, "null argument"); });
  if (rc != B2M_OK) return rc;
  return b2m_verify_batch(vk, 1, &public_input, &n_input, &proof, &proof_len, rng, ok);
}

int b2m_verify_timings(const b2m_vk* vk, char* json, size_t cap) {
  return guard([&] {
    B2M_REQUIRE(vk && json && cap > 0, B2M_ERR_INVALID_ARG, "null argument");
    snprintf(json, cap, "%s", vk->impl->timings_json.c_str());
  });
}

}  // extern "C"
