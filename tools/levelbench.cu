// Register-only ceilings of the batched-affine level arithmetic (no memory traffic): how fast can the addition pass, the
// denominator pass and the inversion run on the whole chip at 1..4 resident CTAs (of 128 threads) per SM?
// Compares with tools/microbench.cu's chained Fq multiplication and XYZZ mixed addition rates.
#include <cstdio>
#include <cuda_runtime.h>
#include "../marlin_b200/csrc/msm_affine.cuh"
using namespace b2m;
typedef FqBls Fq;

// addition pass, plain form: per output dinv = inv * pf, inv *= den, lam, lam^2, y3 (5 multiplications + 6 subtractions)
template <int MINB>
__global__ void __launch_bounds__(128, MINB) pass2_plain(Fq* io, int iters) {
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  Affine<Fq> P{io[t & 1023], io[(t + 1) & 1023]}, Q{io[(t + 2) & 1023], io[(t + 3) & 1023]};
  Fq inv = io[(t + 4) & 1023], pf = io[(t + 5) & 1023];
  for (int i = 0; i < iters; i++) {
    const bool fast = aff_fast(1u, P.x, Q.x);
    const Fq d = Q.x - P.x;
    const Fq den = fast ? d : Fq::one();
    const Fq dinv = inv * pf;
    inv = inv * den;
    const Fq lam = (Q.y - P.y) * dinv;
    Affine<Fq> R;
    R.x = lam.sqr() - P.x - Q.x;
    R.y = lam * (P.x - R.x) - P.y;
    if (!fast) R = aff_add_slow(P, Q, 1u);
    // next operands depend on the result so nothing can be hoisted (stands in for freshly loaded points)
    Q = P; P = R; pf = pf + R.x;
  }
  if (inv.is_zero()) io[t & 1023] = P.x + Q.y;
}
// addition pass, software-pipelined form (two streams)
template <int MINB>
__global__ void __launch_bounds__(128, MINB) pass2_pipe(Fq* io, int iters) {
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  Affine<Fq> P_c{io[t & 1023], io[(t + 1) & 1023]}, Q_c{io[(t + 2) & 1023], io[(t + 3) & 1023]};
  Affine<Fq> P_n{io[(t + 6) & 1023], io[(t + 7) & 1023]}, Q_n{io[(t + 8) & 1023], io[(t + 9) & 1023]};
  Fq inv = io[(t + 4) & 1023], pf = io[(t + 5) & 1023], dinv_c = io[(t + 10) & 1023];
  bool fast_c = true;
  for (int i = 0; i < iters; i++) {
    const Fq lam = (Q_c.y - P_c.y) * dinv_c;
    Affine<Fq> R;
    R.x = lam.sqr() - P_c.x - Q_c.x;
    R.y = lam * (P_c.x - R.x) - P_c.y;
    const bool fast_n = aff_fast(1u, P_n.x, Q_n.x);
    const Fq d = Q_n.x - P_n.x;
    const Fq den = fast_n ? d : Fq::one();
    const Fq dinv_n = inv * pf;
    inv = inv * den;
    if (!fast_c) R = aff_add_slow(P_c, Q_c, 1u);
    P_c = P_n; Q_c = Q_n; fast_c = fast_n; dinv_c = dinv_n;
    Q_n = P_n; P_n = R; pf = pf + R.y;
  }
  if (inv.is_zero()) io[t & 1023] = P_c.x + Q_c.y + dinv_c;
}
// denominator pass: den = x2 - x1, run *= den
template <int MINB>
__global__ void __launch_bounds__(128, MINB) pass1(Fq* io, int iters) {
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  Fq x1 = io[t & 1023], x2 = io[(t + 1) & 1023], run = io[(t + 2) & 1023];
  for (int i = 0; i < iters; i++) {
    const Fq d = x2 - x1;
    const Fq den = aff_fast(1u, x1, x2) ? d : Fq::one();
    run = run * den;
    x1 = x2; x2 = x2 + run;
  }
  if (run.is_zero()) io[t & 1023] = run;
}
template <int MINB>
__global__ void __launch_bounds__(128, MINB) inverses(Fq* io, int iters) {
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  Fq a = io[t & 1023];
  a.l[0] ^= (uint32_t)t * 2654435761u;  // different trip counts per lane, like real data
  a.l[11] &= 0x0fffffffu;
  for (int i = 0; i < iters; i++) a = a.inverse_fast() + Fq::one();
  if (a.is_zero()) io[t & 1023] = a;
}
template <class K>
float time_kernel(K k, int grid, Fq* buf, int iters) {
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  k<<<grid, 128>>>(buf, iters); cudaDeviceSynchronize();
  float best = 1e30f;
  for (int r = 0; r < 3; r++) {
    cudaEventRecord(e0); k<<<grid, 128>>>(buf, iters); cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1); if (ms < best) best = ms;
  }
  return best;
}
int main() {
  cudaDeviceProp prop; cudaGetDeviceProperties(&prop, 0);
  int sms = prop.multiProcessorCount;
  Fq* buf; cudaMalloc(&buf, 1 << 20);
  // valid field elements: small values in Montgomery-agnostic form
  { uint32_t* h = (uint32_t*)malloc(1 << 20); for (int i = 0; i < (1 << 18); i++) h[i] = (i % 12 == 11) ? 0x0a0111eau : (uint32_t)(i * 2654435761u + 12345u);
    cudaMemcpy(buf, h, 1 << 20, cudaMemcpyHostToDevice); free(h); }
  printf("{\"device\": \"%s\", \"sms\": %d", prop.name, sms);
  const int it = 400;
#define RUN(name, kern, bps, units)                                                                    \
  { float ms = time_kernel(kern<bps>, sms * bps, buf, it);                                              \
    printf(", \"%s_bps%d_G_per_s\": %.3f", name, bps, (double)sms * bps * 128 * it * units / ms / 1e6); }
  RUN("pass2_plain_adds", pass2_plain, 1, 1) RUN("pass2_plain_adds", pass2_plain, 2, 1) RUN("pass2_plain_adds", pass2_plain, 3, 1) RUN("pass2_plain_adds", pass2_plain, 4, 1)
  RUN("pass2_pipe_adds", pass2_pipe, 1, 1) RUN("pass2_pipe_adds", pass2_pipe, 2, 1) RUN("pass2_pipe_adds", pass2_pipe, 3, 1) RUN("pass2_pipe_adds", pass2_pipe, 4, 1)
  RUN("pass1_muls", pass1, 1, 1) RUN("pass1_muls", pass1, 2, 1) RUN("pass1_muls", pass1, 4, 1) RUN("pass1_muls", pass1, 6, 1)
  { float ms = time_kernel(inverses<4>, sms * 4, buf, 8); printf(", \"inverse_fast_bps4_M_per_s\": %.2f", (double)sms * 4 * 128 * 8 / ms / 1e3); }
  { float ms = time_kernel(inverses<8>, sms * 8, buf, 8); printf(", \"inverse_fast_bps8_M_per_s\": %.2f", (double)sms * 8 * 128 * 8 / ms / 1e3); }
  printf("}\n");
  return 0;
}
