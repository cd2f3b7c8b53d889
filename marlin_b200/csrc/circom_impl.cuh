// Kernels and chunked host drivers of circom.cuh.
//
// Constraint decoding: the section is copied to the device in chunks of whole constraints holding at most ARK_DECODE_CHUNK
// terms (or one constraint, when a single constraint holds more) and at most CIRCOM_CHUNK_ROWS constraints, so device
// scratch stays bounded whatever the file size.  Per chunk and matrix:
//   1. one thread per term reads its (u32 wire, 32-byte coefficient) entry, checks wire < nWires and coefficient < r
//      (the lowest bad term of the chunk, in file order, goes through atomicMin), converts to Montgomery form, shifts the
//      column past the instance padding and flags its row when the row is not strictly ascending or holds a zero;
//   2. one block per flagged row sorts the row by column (a bitonic network in global memory, so a row of any length
//      fits), then sums equal columns and drops zero sums;
//   3. the row lengths are scanned (scan.cuh) into row pointers and the rows compacted.
// Every term's byte offset follows from the term-count prefix sums: LC j of constraint k starts at
// 4 (3k + j) + 36 (terms before it), so the host walk's three row-pointer arrays are all the kernel needs.
//
// Satisfiability: z is uploaded once, rows follow in chunks of at most ARK_DECODE_CHUNK entries per matrix; spmv_kernel
// (poly_impl.cuh) gives <M_r, z> for the three matrices and one thread per row compares; the lowest failing row goes
// through atomicMin, and the first chunk holding one stops the call.
#pragma once
#include <algorithm>
#include <vector>

#include "ark_points.cuh"
#include "circom.cuh"
#include "devmem.cuh"
#include "poly_impl.cuh"
#include "scan.cuh"

namespace b2m {

constexpr size_t CIRCOM_CHUNK_ROWS = ARK_DECODE_CHUNK;
constexpr int CIRCOM_SORT_THREADS = 128;

// the row k of chunk-local rows [0, mc) holding absolute term g: rp[k] <= g < rp[k + 1]
__device__ __forceinline__ uint32_t circom_row_of(const uint64_t* rp, uint32_t mc, uint64_t g) {
  uint32_t lo = 0, hi = mc;
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) / 2;
    if (rp[mid] <= g) lo = mid;
    else hi = mid;
  }
  return lo;
}

// One thread per term of matrix j in the chunk.  bytes: the chunk's constraints (4-byte aligned: every field of the
// section sits at a multiple of 4 from the chunk start); rp0..rp2: row pointers of the chunk's mc + 1 rows, absolute.
template <class Fr>
__global__ void circom_decode_kernel(const uint8_t* bytes, uint64_t sec_off, const uint64_t* rp0, const uint64_t* rp1, const uint64_t* rp2, int j,
                                     uint32_t mc, size_t nt, uint64_t n_wires, uint64_t ni0, uint64_t shift, uint64_t* col, Fr* coeff,
                                     uint32_t* row_of, uint32_t* flag, uint32_t* any, unsigned long long* first_bad) {
  const size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (t >= nt) return;
  const uint64_t* rp = j == 0 ? rp0 : j == 1 ? rp1 : rp2;
  const uint64_t g = rp[0] + t;
  const uint32_t k = circom_row_of(rp, mc, g);
  uint64_t before = (rp0[k] - rp0[0]) + (rp1[k] - rp1[0]) + (rp2[k] - rp2[0]);
  if (j > 0) before += rp0[k + 1] - rp0[k];
  if (j > 1) before += rp1[k + 1] - rp1[k];
  const uint64_t i = g - rp[k];
  const size_t at = 4 * (3 * (size_t)k + j) + CIRCOM_TERM_BYTES * (before + i) + 4;
  const uint32_t* w = reinterpret_cast<const uint32_t*>(bytes + at);
  const uint32_t wire = w[0];
  Fr c;
#pragma unroll
  for (int l = 0; l < Fr::N; l++) c.l[l] = w[1 + l];
  bool below = false;  // c < r, decided at the highest limb where the two differ
#pragma unroll
  for (int l = Fr::N - 1; l >= 0; l--) {
    const uint32_t m = Fr::Params::mod(l);
    if (c.l[l] != m) {
      below = c.l[l] < m;
      break;
    }
  }
  row_of[t] = k;
  const int reason = wire >= n_wires ? 1 : !below ? 2 : 0;
  if (reason) {
    atomicMin(first_bad, (unsigned long long)(((sec_off + at) << 2) | (uint64_t)reason));
    col[t] = 0;
    st_fr(coeff + t, Fr::zero());
    return;
  }
  col[t] = wire < ni0 ? wire : wire + shift;
  st_fr(coeff + t, Fr::from_canonical(c));
  // the previous term's wire is 9 words back; the column shift keeps the order of wires
  if (c.is_zero() || (i > 0 && w[-9] >= wire)) {
    flag[k] = 1;
    *any = 1;
  }
}

template <class Fr>
__device__ __forceinline__ void circom_swap(uint64_t* c, Fr* v, size_t a, size_t b) {
  const uint64_t tc = c[a];
  c[a] = c[b];
  c[b] = tc;
  const Fr tv = ld_fr(v + a);
  st_fr(v + a, ld_fr(v + b));
  st_fr(v + b, tv);
}

// One block per row of the chunk; rows that are not flagged return at once.  The sort is the bitonic network in its
// single-direction form (each merge starts with a mirrored comparison), so positions past the row's length act as +inf
// and never move: a row of any length sorts in place.  One thread then sums equal columns and drops zero sums.
template <class Fr>
__global__ void __launch_bounds__(CIRCOM_SORT_THREADS) circom_normalise_kernel(const uint64_t* rp, const uint32_t* flag, uint64_t* col, Fr* coeff,
                                                                               uint32_t* len) {
  const uint32_t k = blockIdx.x;
  if (!flag[k]) return;
  const size_t s = rp[k] - rp[0], n = rp[k + 1] - rp[k];
  uint64_t* c = col + s;
  Fr* v = coeff + s;
  size_t P = 1;
  while (P < n) P <<= 1;
  for (size_t size = 2; size <= P; size <<= 1) {
    for (size_t half = size / 2; half >= 1; half >>= 1) {
      for (size_t q = threadIdx.x; q < P / 2; q += blockDim.x) {
        const size_t blk = q / half, off = q % half;
        const size_t a = blk * 2 * half + off;
        const size_t b = half == size / 2 ? blk * 2 * half + 2 * half - 1 - off : a + half;
        if (b < n && c[a] > c[b]) circom_swap(c, v, a, b);
      }
      __syncthreads();
    }
  }
  if (threadIdx.x != 0) return;
  size_t w = 0;
  for (size_t i = 0; i < n;) {
    const uint64_t ci = c[i];
    Fr acc = ld_fr(v + i);
    for (i++; i < n && c[i] == ci; i++) acc = acc + ld_fr(v + i);
    if (!acc.is_zero()) {
      c[w] = ci;
      st_fr(v + w, acc);
      w++;
    }
  }
  len[k] = (uint32_t)w;
}

static __global__ void circom_row_len_kernel(const uint64_t* rp, uint32_t mc, uint32_t* len) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k <= mc) len[k] = k < mc ? (uint32_t)(rp[k + 1] - rp[k]) : 0u;
}

template <class Fr>
__global__ void circom_compact_kernel(const uint64_t* rp, size_t nt, const uint32_t* row_of, const uint32_t* len, const uint32_t* start,
                                      const uint64_t* col, const Fr* coeff, uint64_t* out_col, Fr* out_coeff) {
  const size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (t >= nt) return;
  const uint32_t k = row_of[t];
  const uint64_t i = rp[0] + t - rp[k];
  if (i >= len[k]) return;
  const size_t o = start[k] + i;
  out_col[o] = col[t];
  st_fr(out_coeff + o, ld_fr(coeff + t));
}

static __global__ void circom_row_ptr_kernel(const uint32_t* start, uint32_t mc, uint64_t base, uint64_t* out) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k <= mc) out[k] = base + start[k];
}

template <class Fr>
CircomBad circom_decode_constraints(Ctx& cx, const uint8_t* bytes, size_t len, size_t m, const uint64_t* const* row_ptrs, uint64_t n_wires,
                                    uint64_t ni0, uint64_t shift, uint64_t* const* out_row_ptr, uint64_t* const* out_col, uint64_t* const* out_coeff) {
  static_assert(sizeof(Fr) == 32, "circom coefficients are 32 bytes (n8 = 32)");
  for (int j = 0; j < 3; j++) out_row_ptr[j][0] = 0;
  if (m == 0) return CircomBad{0, 0, 0};
  const uint64_t* const* rp = row_ptrs;
  auto total = [&](size_t k) { return rp[0][k] + rp[1][k] + rp[2][k]; };
  auto offset = [&](size_t k) { return 12 * k + CIRCOM_TERM_BYTES * total(k); };  // byte offset of constraint k
  for (int j = 0; j < 3; j++) B2M_REQUIRE(rp[j][0] == 0, B2M_ERR_INVALID_ARG, "row_ptrs[%d][0] is not 0", j);
  B2M_REQUIRE(offset(m) <= len, B2M_ERR_INVALID_ARG, "the row pointers describe %llu bytes, the section has %zu", (unsigned long long)offset(m), len);
  B2M_REQUIRE(n_wires <= 0xffffffffull && ni0 <= n_wires, B2M_ERR_INVALID_ARG, "n_wires %llu / ni0 %llu", (unsigned long long)n_wires,
              (unsigned long long)ni0);

  // chunks of whole constraints
  std::vector<size_t> cuts{0};
  size_t max_terms = 1, max_rows = 1;
  while (cuts.back() < m) {
    const size_t k0 = cuts.back();
    size_t a = k0 + 1, b = std::min(m, k0 + CIRCOM_CHUNK_ROWS);
    while (a < b) {
      const size_t mid = (a + b + 1) / 2;
      if (total(mid) - total(k0) <= ARK_DECODE_CHUNK) a = mid;
      else b = mid - 1;
    }
    cuts.push_back(a);
    max_terms = std::max<size_t>(max_terms, total(a) - total(k0));
    max_rows = std::max(max_rows, a - k0);
  }
  B2M_REQUIRE(max_terms <= 0xffffffffull, B2M_ERR_UNSUPPORTED, "a constraint of %zu terms", max_terms);
  const size_t R = max_rows + 1;
  DBuf<uint8_t> dbytes(cx, 12 * max_rows + CIRCOM_TERM_BYTES * max_terms);
  DBuf<uint64_t> drp(cx, 3 * R), dcol(cx, max_terms), docol(cx, max_terms), dorp(cx, 3 * R);
  DBuf<Fr> dcoeff(cx, max_terms), docoeff(cx, max_terms);
  DBuf<uint32_t> drow(cx, max_terms), dflag(cx, 3 * R), dlen(cx, R), dstart(cx, R), dany(cx, 3);
  DBuf<unsigned long long> dbad(cx, 1);

  for (size_t c = 0; c + 1 < cuts.size(); c++) {
    const size_t k0 = cuts[c], k1 = cuts[c + 1];
    const uint32_t mc = (uint32_t)(k1 - k0);
    size_t nt[3], tb[3];
    for (int j = 0; j < 3; j++) {
      nt[j] = rp[j][k1] - rp[j][k0];
      tb[j] = j == 0 ? 0 : tb[j - 1] + nt[j - 1];
    }
    size_t sp = cx.span_begin("circom_h2d", (double)(tb[2] + nt[2]));
    dbytes.upload(bytes + offset(k0), offset(k1) - offset(k0));
    for (int j = 0; j < 3; j++) B2M_CUDA(cudaMemcpyAsync(drp.p + j * R, rp[j] + k0, (mc + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, cx.stream));
    cx.span_end(sp);
    sp = cx.span_begin("circom_decode", (double)(tb[2] + nt[2]));
    B2M_CUDA(cudaMemsetAsync(dbad.p, 0xff, sizeof(unsigned long long), cx.stream));
    B2M_CUDA(cudaMemsetAsync(dany.p, 0, 3 * sizeof(uint32_t), cx.stream));
    B2M_CUDA(cudaMemsetAsync(dflag.p, 0, 3 * R * sizeof(uint32_t), cx.stream));
    for (int j = 0; j < 3; j++) {
      if (!nt[j]) continue;
      circom_decode_kernel<Fr><<<div_up(nt[j], 256), 256, 0, cx.stream>>>(dbytes.p, offset(k0), drp.p, drp.p + R, drp.p + 2 * R, j, mc, nt[j], n_wires,
                                                                         ni0, shift, dcol.p + tb[j], dcoeff.p + tb[j], drow.p + tb[j], dflag.p + j * R,
                                                                         dany.p + j, dbad.p);
      B2M_CHECK_LAUNCH();
      cx.launches++;
    }
    unsigned long long bad = 0;
    dbad.download(&bad, 1);
    if (bad != ~0ull) {
      cx.span_end(sp);
      const uint64_t off = bad >> 2;
      size_t lo = k0, hi = k1;  // the constraint: the last k with offset(k) <= off
      while (hi - lo > 1) {
        const size_t mid = (lo + hi) / 2;
        if (offset(mid) <= off) lo = mid;
        else hi = mid;
      }
      const size_t k = lo;
      uint64_t lc = offset(k);
      for (int j = 0; j < 3; j++) {
        const uint64_t n = rp[j][k + 1] - rp[j][k];
        if (off < lc + 4 + CIRCOM_TERM_BYTES * n) return CircomBad{j, (size_t)(rp[j][k] + (off - lc - 4) / CIRCOM_TERM_BYTES), (int)(bad & 3)};
        lc += 4 + CIRCOM_TERM_BYTES * n;
      }
      throw Error(B2M_ERR_INVALID_ARG, fmt("bad term at byte %llu is in no matrix", (unsigned long long)off));
    }
    uint32_t any[3];
    dany.download(any, 3);
    for (int j = 0; j < 3; j++) {
      const uint64_t* drpj = drp.p + j * R;
      circom_row_len_kernel<<<div_up(mc + 1, 256), 256, 0, cx.stream>>>(drpj, mc, dlen.p);
      B2M_CHECK_LAUNCH();
      cx.launches++;
      if (any[j]) {
        circom_normalise_kernel<Fr><<<mc, CIRCOM_SORT_THREADS, 0, cx.stream>>>(drpj, dflag.p + j * R, dcol.p + tb[j], dcoeff.p + tb[j], dlen.p);
        B2M_CHECK_LAUNCH();
        cx.launches++;
      }
      exclusive_scan_u32(cx, dlen.p, dstart.p, mc + 1);
      if (nt[j]) {
        circom_compact_kernel<Fr><<<div_up(nt[j], 256), 256, 0, cx.stream>>>(drpj, nt[j], drow.p + tb[j], dlen.p, dstart.p, dcol.p + tb[j],
                                                                            dcoeff.p + tb[j], docol.p + tb[j], docoeff.p + tb[j]);
        B2M_CHECK_LAUNCH();
        cx.launches++;
      }
      circom_row_ptr_kernel<<<div_up(mc + 1, 256), 256, 0, cx.stream>>>(dstart.p, mc, out_row_ptr[j][k0], dorp.p + j * R);
      B2M_CHECK_LAUNCH();
      cx.launches++;
    }
    cx.span_end(sp);
    sp = cx.span_begin("circom_d2h", (double)(tb[2] + nt[2]));
    for (int j = 0; j < 3; j++) {
      const uint64_t base = out_row_ptr[j][k0];
      B2M_CUDA(cudaMemcpyAsync(out_row_ptr[j] + k0, dorp.p + j * R, (mc + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, cx.stream));
      cx.sync();
      const size_t n_out = out_row_ptr[j][k1] - base;
      if (n_out) {
        B2M_CUDA(cudaMemcpyAsync(out_col[j] + base, docol.p + tb[j], n_out * sizeof(uint64_t), cudaMemcpyDeviceToHost, cx.stream));
        B2M_CUDA(cudaMemcpyAsync(out_coeff[j] + 4 * base, docoeff.p + tb[j], n_out * sizeof(Fr), cudaMemcpyDeviceToHost, cx.stream));
      }
    }
    cx.sync();
    cx.span_end(sp);
  }
  return CircomBad{0, 0, 0};
}

// ---- satisfiability ---------------------------------------------------------------------------------------------------
// rows [0, rows] of a chunk's row pointers and its ne entries' columns, narrowed to the u32 form spmv_kernel reads; a
// column >= nv goes through atomicMin and reads z[0] instead
static __global__ void r1cs_narrow_kernel(const uint64_t* rp, size_t rows, const uint64_t* col, size_t ne, uint64_t nv, uint32_t* rp32, uint32_t* col32,
                                          unsigned long long* bad_col) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i <= rows) rp32[i] = (uint32_t)(rp[i] - rp[0]);
  if (i < ne) {
    uint64_t c = col[i];
    if (c >= nv) {
      atomicMin(bad_col, (unsigned long long)i);
      c = 0;
    }
    col32[i] = (uint32_t)c;
  }
}

template <class Fr>
__global__ void r1cs_rows_kernel(const Fr* az, const Fr* bz, const Fr* cz, size_t rows, size_t r0, unsigned long long* bad) {
  const size_t r = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (r >= rows) return;
  if (ld_fr(az + r) * ld_fr(bz + r) != ld_fr(cz + r)) atomicMin(bad, (unsigned long long)(r0 + r));
}

template <class Fr>
size_t r1cs_check(Ctx& cx, size_t nc, size_t nv, size_t ni, const b2m_matrix* const* mats, const uint64_t* instance, const uint64_t* witness) {
  B2M_REQUIRE(ni >= 1 && ni <= nv && nv <= 0xffffffffull, B2M_ERR_INVALID_ARG, "num_instance %zu, num_variables %zu", ni, nv);
  if (nc == 0) return 0;
  for (int j = 0; j < 3; j++) {
    const uint64_t* rp = mats[j]->row_ptr;
    B2M_REQUIRE(rp[0] == 0, B2M_ERR_INVALID_ARG, "matrix %c: row_ptr[0] is not 0", "ABC"[j]);
    for (size_t r = 0; r < nc; r++)
      B2M_REQUIRE(rp[r + 1] >= rp[r], B2M_ERR_INVALID_ARG, "matrix %c: row_ptr[%zu] < row_ptr[%zu]", "ABC"[j], r + 1, r);
  }
  DBuf<Fr> z(cx, nv);
  z.upload(reinterpret_cast<const Fr*>(instance), ni);
  if (nv > ni) B2M_CUDA(cudaMemcpyAsync(z.p + ni, witness, (nv - ni) * sizeof(Fr), cudaMemcpyHostToDevice, cx.stream));

  // chunks of whole rows with at most ARK_DECODE_CHUNK entries per matrix (or one row)
  auto nnz = [&](int j, size_t r0, size_t r1) { return mats[j]->row_ptr[r1] - mats[j]->row_ptr[r0]; };
  std::vector<size_t> cuts{0};
  size_t max_ne = 1, max_rows = 1;
  while (cuts.back() < nc) {
    const size_t r0 = cuts.back();
    size_t a = r0 + 1, b = std::min(nc, r0 + CIRCOM_CHUNK_ROWS);
    while (a < b) {
      const size_t mid = (a + b + 1) / 2;
      if (std::max({nnz(0, r0, mid), nnz(1, r0, mid), nnz(2, r0, mid)}) <= ARK_DECODE_CHUNK) a = mid;
      else b = mid - 1;
    }
    cuts.push_back(a);
    for (int j = 0; j < 3; j++) max_ne = std::max<size_t>(max_ne, nnz(j, r0, a));
    max_rows = std::max(max_rows, a - r0);
  }
  B2M_REQUIRE(max_ne <= 0xffffffffull, B2M_ERR_UNSUPPORTED, "a row of %zu entries", max_ne);
  DBuf<uint64_t> drp(cx, max_rows + 1), dcol(cx, max_ne);
  DBuf<uint32_t> drp32(cx, max_rows + 1), dcol32(cx, max_ne);
  DBuf<Fr> dcoeff(cx, max_ne), dout(cx, 3 * max_rows);
  DBuf<unsigned long long> dbad(cx, 2);  // lowest failing row, lowest column out of range
  for (size_t c = 0; c + 1 < cuts.size(); c++) {
    const size_t r0 = cuts[c], r1 = cuts[c + 1], rows = r1 - r0;
    B2M_CUDA(cudaMemsetAsync(dbad.p, 0xff, 2 * sizeof(unsigned long long), cx.stream));
    for (int j = 0; j < 3; j++) {
      const b2m_matrix* mt = mats[j];
      const size_t e0 = mt->row_ptr[r0], ne = nnz(j, r0, r1);
      size_t sp = cx.span_begin("r1cs_check_h2d", (double)ne);
      drp.upload(mt->row_ptr + r0, rows + 1);
      if (ne) {
        dcol.upload(mt->col + e0, ne);
        dcoeff.upload(reinterpret_cast<const Fr*>(mt->coeff) + e0, ne);
      }
      cx.span_end(sp);
      sp = cx.span_begin("r1cs_check", (double)ne);
      r1cs_narrow_kernel<<<div_up(std::max(rows + 1, ne), 256), 256, 0, cx.stream>>>(drp.p, rows, dcol.p, ne, nv, drp32.p, dcol32.p, dbad.p + 1);
      B2M_CHECK_LAUNCH();
      spmv_kernel<Fr><<<div_up(rows, 256), 256, 0, cx.stream>>>(drp32.p, dcol32.p, dcoeff.p, z.p, rows, dout.p + j * max_rows);
      B2M_CHECK_LAUNCH();
      cx.launches += 2;
      unsigned long long bad_col = 0;
      B2M_CUDA(cudaMemcpyAsync(&bad_col, dbad.p + 1, sizeof(bad_col), cudaMemcpyDeviceToHost, cx.stream));
      cx.sync();
      cx.span_end(sp);
      if (bad_col != ~0ull) {
        const size_t e = e0 + (size_t)bad_col;
        const size_t r = (size_t)(std::upper_bound(mt->row_ptr, mt->row_ptr + nc + 1, (uint64_t)e) - mt->row_ptr) - 1;
        throw Error(B2M_ERR_INVALID_ARG, fmt("matrix %c row %zu: column %llu >= num_variables %zu", "ABC"[j], r, (unsigned long long)mt->col[e], nv));
      }
    }
    r1cs_rows_kernel<Fr><<<div_up(rows, 256), 256, 0, cx.stream>>>(dout.p, dout.p + max_rows, dout.p + 2 * max_rows, rows, r0, dbad.p);
    B2M_CHECK_LAUNCH();
    cx.launches++;
    unsigned long long bad = 0;
    dbad.download(&bad, 1);
    if (bad != ~0ull) return (size_t)bad;
  }
  return nc;
}

#define B2M_INSTANTIATE_CIRCOM(FR)                                                                                                     \
  template CircomBad circom_decode_constraints<FR>(Ctx&, const uint8_t*, size_t, size_t, const uint64_t* const*, uint64_t, uint64_t, uint64_t, \
                                                   uint64_t* const*, uint64_t* const*, uint64_t* const*);                             \
  template size_t r1cs_check<FR>(Ctx&, size_t, size_t, size_t, const b2m_matrix* const*, const uint64_t*, const uint64_t*);

}  // namespace b2m
