// Kernels and chunked host drivers of ark_points.cuh.  One thread per point (or Fr element).  Each decode kernel writes the point, its
// status, and folds the index of every invalid point into one device word with atomicMin; chunks run in file order and the
// driver stops at the first chunk with a failure, so the index it reports is the lowest invalid one of the whole input.
#pragma once
#include <algorithm>

#include "ark_points.cuh"
#include "curve.cuh"
#include "devmem.cuh"
#include "g1_decode.cuh"
#include "g2_decode.cuh"

namespace b2m {

// one instantiation per form: the two paths together would not fit the register file
template <class Fq, bool compressed>
__global__ void g1_decode_ark_kernel(const uint8_t* bytes, size_t n, Affine<Fq>* out, int* status, unsigned long long* first_bad) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<Fq> p;
  const int s = compressed ? g1_decompress<Fq>(bytes + i * (Fq::N * 4), &p) : g1_decode_uncompressed<Fq>(bytes + i * (Fq::N * 8), &p);
  out[i] = p;
  status[i] = s;
  if (s != G1_OK) atomicMin(first_bad, (unsigned long long)i);
}

template <class Fq, bool compressed>
__global__ void g2_decode_ark_kernel(const uint8_t* bytes, size_t n, uint8_t* out, int* status, unsigned long long* first_bad) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int s = g2_decode<Fq>(bytes + i * (compressed ? Fq::N * 8 : Fq::N * 16), compressed, out + i * (Fq::N * 16));
  status[i] = s;
  if (s != G1_OK) atomicMin(first_bad, (unsigned long long)i);
}

// snarkjs LEM points (.ptau files): a form of their own, so the ark kernels above keep their register allocation
template <class Fq>
__global__ void g1_decode_lem_kernel(const uint8_t* bytes, size_t n, Affine<Fq>* out, int* status, unsigned long long* first_bad) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<Fq> p;
  const int s = g1_decode_lem<Fq>(bytes + i * (Fq::N * 8), &p);
  out[i] = p;
  status[i] = s;
  if (s != G1_OK) atomicMin(first_bad, (unsigned long long)i);
}

template <class Fq>
__global__ void g2_decode_lem_kernel(const uint8_t* bytes, size_t n, uint8_t* out, int* status, unsigned long long* first_bad) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int s = g2_decode_lem<Fq>(bytes + i * (Fq::N * 16), out + i * (Fq::N * 16));
  status[i] = s;
  if (s != G1_OK) atomicMin(first_bad, (unsigned long long)i);
}

template <class Fq>
__global__ void g1_compress_kernel(const Affine<Fq>* in, size_t n, uint8_t* out) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  g1_compress<Fq>(in[i], out + i * (Fq::N * 4));
}

// Shared chunk loop: in_bytes / out_bytes per point; launch(din, m, dout, dstatus, dbad) issues the kernel of one chunk.
template <class Launch>
ArkBad ark_decode_chunks(Ctx& cx, const uint8_t* bytes, size_t n, size_t in_bytes, uint8_t* out, size_t out_bytes, const char* kernel_name,
                         Launch launch) {
  const size_t chunk = std::min(n, ARK_DECODE_CHUNK);
  DBuf<uint8_t> din(cx, chunk * in_bytes), dout(cx, chunk * out_bytes);
  DBuf<int> dstatus(cx, chunk);
  DBuf<unsigned long long> dbad(cx, 1);
  for (size_t at = 0; at < n; at += chunk) {
    const size_t m = std::min(chunk, n - at);
    B2M_CUDA(cudaMemsetAsync(dbad.p, 0xff, sizeof(unsigned long long), cx.stream));
    size_t sp = cx.span_begin("ark_h2d", (double)m);
    din.upload(bytes + at * in_bytes, m * in_bytes);
    cx.span_end(sp);
    sp = cx.span_begin(kernel_name, (double)m);
    launch(din.p, m, dout.p, dstatus.p, dbad.p);
    B2M_CHECK_LAUNCH();
    cx.launches++;
    cx.span_end(sp);
    unsigned long long bad = 0;
    dbad.download(&bad, 1);
    if (bad != ~0ull) {
      int reason = 0;
      B2M_CUDA(cudaMemcpyAsync(&reason, dstatus.p + bad, sizeof(int), cudaMemcpyDeviceToHost, cx.stream));
      cx.sync();
      return ArkBad{at + (size_t)bad, reason};
    }
    sp = cx.span_begin("ark_d2h", (double)m);
    dout.download(out + at * out_bytes, m * out_bytes);
    cx.span_end(sp);
  }
  return ArkBad{n, G1_OK};
}

template <class Fq>
ArkBad g1_decode_ark(Ctx& cx, const uint8_t* bytes, size_t n, bool compressed, uint64_t* out_xy) {
  return ark_decode_chunks(cx, bytes, n, compressed ? Fq::N * 4 : Fq::N * 8, reinterpret_cast<uint8_t*>(out_xy), sizeof(Affine<Fq>),
                           "ark_g1_decode", [&](const uint8_t* din, size_t m, uint8_t* dout, int* st, unsigned long long* bad) {
                             Affine<Fq>* o = reinterpret_cast<Affine<Fq>*>(dout);
                             if (compressed) g1_decode_ark_kernel<Fq, true><<<div_up(m, 128), 128, 0, cx.stream>>>(din, m, o, st, bad);
                             else g1_decode_ark_kernel<Fq, false><<<div_up(m, 128), 128, 0, cx.stream>>>(din, m, o, st, bad);
                           });
}

template <class Fq>
ArkBad g2_decode_ark(Ctx& cx, const uint8_t* bytes, size_t n, bool compressed, uint8_t* out) {
  return ark_decode_chunks(cx, bytes, n, compressed ? Fq::N * 8 : Fq::N * 16, out, Fq::N * 16, "ark_g2_decode",
                           [&](const uint8_t* din, size_t m, uint8_t* dout, int* st, unsigned long long* bad) {
                             if (compressed) g2_decode_ark_kernel<Fq, true><<<div_up(m, 128), 128, 0, cx.stream>>>(din, m, dout, st, bad);
                             else g2_decode_ark_kernel<Fq, false><<<div_up(m, 128), 128, 0, cx.stream>>>(din, m, dout, st, bad);
                           });
}

template <class Fq>
ArkBad g1_decode_lem_points(Ctx& cx, const uint8_t* bytes, size_t n, uint64_t* out_xy) {
  return ark_decode_chunks(cx, bytes, n, Fq::N * 8, reinterpret_cast<uint8_t*>(out_xy), sizeof(Affine<Fq>), "lem_g1_decode",
                           [&](const uint8_t* din, size_t m, uint8_t* dout, int* st, unsigned long long* bad) {
                             g1_decode_lem_kernel<Fq><<<div_up(m, 128), 128, 0, cx.stream>>>(din, m, reinterpret_cast<Affine<Fq>*>(dout), st, bad);
                           });
}

template <class Fq>
ArkBad g2_decode_lem_points(Ctx& cx, const uint8_t* bytes, size_t n, uint8_t* out) {
  return ark_decode_chunks(cx, bytes, n, Fq::N * 16, out, Fq::N * 16, "lem_g2_decode",
                           [&](const uint8_t* din, size_t m, uint8_t* dout, int* st, unsigned long long* bad) {
                             g2_decode_lem_kernel<Fq><<<div_up(m, 128), 128, 0, cx.stream>>>(din, m, dout, st, bad);
                           });
}

template <class Fq>
void g1_to_compressed(Ctx& cx, const uint64_t* points_xy, size_t n, uint8_t* out) {
  const size_t chunk = std::min(n, ARK_DECODE_CHUNK * 4);
  DBuf<Affine<Fq>> din(cx, chunk);
  DBuf<uint8_t> dout(cx, chunk * Fq::N * 4);
  for (size_t at = 0; at < n; at += chunk) {
    const size_t m = std::min(chunk, n - at);
    din.upload(reinterpret_cast<const Affine<Fq>*>(points_xy) + at, m);
    g1_compress_kernel<Fq><<<div_up(m, 256), 256, 0, cx.stream>>>(din.p, m, dout.p);
    B2M_CHECK_LAUNCH();
    cx.launches++;
    dout.download(out + at * Fq::N * 4, m * Fq::N * 4);
  }
}

// ---- Fr elements ------------------------------------------------------------------------------------------------------
// One thread per element: canonical bytes (staged in device memory) -> check < r -> Montgomery.  `base` is the index of
// the chunk's first element in the whole input, so one atomicMin word holds the lowest bad index across every chunk.
template <class Fr>
__global__ void fr_decode_ark_kernel(const uint8_t* bytes, size_t n, size_t base, Fr* out, unsigned long long* first_bad) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  Fr c = ld_fr(reinterpret_cast<const Fr*>(bytes) + i);
  bool below = false;  // c < r, decided at the highest limb where the two differ (c == r is not below)
#pragma unroll
  for (int k = Fr::N - 1; k >= 0; k--) {
    const uint32_t m = Fr::Params::mod(k);
    if (c.l[k] != m) {
      below = c.l[k] < m;
      break;
    }
  }
  if (!below) {
    atomicMin(first_bad, (unsigned long long)(base + i));
    st_fr(out + i, Fr::zero());
    return;
  }
  st_fr(out + i, Fr::from_canonical(c));
}

template <class Fr>
__global__ void fr_to_canonical_kernel(const Fr* in, size_t n, Fr* out) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  st_fr(out + i, ld_fr(in + i).to_canonical());
}

template <class Fr>
ArkBad fr_decode_ark(Ctx& cx, const uint8_t* bytes, size_t n, Fr* out_dev) {
  if (n == 0) return ArkBad{0, 0};
  const size_t chunk = std::min(n, ARK_DECODE_CHUNK);
  DBuf<uint8_t> din(cx, chunk * sizeof(Fr));
  DBuf<unsigned long long> dbad(cx, 1);
  B2M_CUDA(cudaMemsetAsync(dbad.p, 0xff, sizeof(unsigned long long), cx.stream));
  for (size_t at = 0; at < n; at += chunk) {
    const size_t m = std::min(chunk, n - at);
    size_t sp = cx.span_begin("ark_h2d", (double)m);
    din.upload(bytes + at * sizeof(Fr), m * sizeof(Fr));
    cx.span_end(sp);
    sp = cx.span_begin("ark_fr_decode", (double)m);
    fr_decode_ark_kernel<Fr><<<div_up(m, 256), 256, 0, cx.stream>>>(din.p, m, at, out_dev + at, dbad.p);
    B2M_CHECK_LAUNCH();
    cx.launches++;
    cx.span_end(sp);
  }
  unsigned long long bad = 0;
  dbad.download(&bad, 1);
  return bad == ~0ull ? ArkBad{n, 0} : ArkBad{(size_t)bad, FR_NOT_CANONICAL};
}

template <class Fr>
void fr_to_canonical(Ctx& cx, const Fr* in_dev, size_t n, uint8_t* out) {
  if (n == 0) return;
  const size_t chunk = std::min(n, ARK_DECODE_CHUNK * 4);
  DBuf<Fr> dout(cx, chunk);
  for (size_t at = 0; at < n; at += chunk) {
    const size_t m = std::min(chunk, n - at);
    fr_to_canonical_kernel<Fr><<<div_up(m, 256), 256, 0, cx.stream>>>(in_dev + at, m, dout.p);
    B2M_CHECK_LAUNCH();
    cx.launches++;
    dout.download(reinterpret_cast<Fr*>(out) + at, m);
  }
}

#define B2M_INSTANTIATE_ARK_POINTS(FQ)                                                                  \
  template ArkBad g1_decode_ark<FQ>(Ctx&, const uint8_t*, size_t, bool, uint64_t*);                  \
  template ArkBad g2_decode_ark<FQ>(Ctx&, const uint8_t*, size_t, bool, uint8_t*);                   \
  template ArkBad g1_decode_lem_points<FQ>(Ctx&, const uint8_t*, size_t, uint64_t*);                         \
  template ArkBad g2_decode_lem_points<FQ>(Ctx&, const uint8_t*, size_t, uint8_t*);                          \
  template void g1_to_compressed<FQ>(Ctx&, const uint64_t*, size_t, uint8_t*);
#define B2M_INSTANTIATE_ARK_FR(FR)                                                                      \
  template ArkBad fr_decode_ark<FR>(Ctx&, const uint8_t*, size_t, FR*);                              \
  template void fr_to_canonical<FR>(Ctx&, const FR*, size_t, uint8_t*);

}  // namespace b2m
