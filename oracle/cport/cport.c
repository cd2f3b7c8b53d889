#include "cport_core.h"

/* ---- MSM ------------------------------------------------------------------------------------------------ */
/* bases: affine x||y Montgomery limbs ((0,0) = infinity); scalars: canonical 4-limb integers; out: affine. */
int cport_msm(int curve, const u64* bases, const u64* scalars, size_t n, u64* out_xy, int threads) {
  init_all();
  if (threads <= 0) threads = max_threads();
  if (curve == 0) { bls_jac r; bls_msm(&r, (const bls_aff*)bases, scalars, n, 255, &BLS_FQ, threads); bls_aff a; bls_to_affine(&a, &r, &BLS_FQ); memcpy(out_xy, &a, sizeof(a)); }
  else { bn_jac r; bn_msm(&r, (const bn_aff*)bases, scalars, n, 254, &BN_FQ, threads); bn_aff a; bn_to_affine(&a, &r, &BN_FQ); memcpy(out_xy, &a, sizeof(a)); }
  return 0;
}
/* distinct cheap bases for timing runs: P_i = (i + 1) * g by incremental addition, batch-free normalisation */
int cport_gen_bases(int curve, const u64* g_xy, size_t n, u64* out) {
  init_all();
  if (curve == 0) {
    bls_aff g; memcpy(&g, g_xy, sizeof(g)); bls_jac acc; bls_jac_set_inf(&acc); bls_aff* o = (bls_aff*)out;
    bls_jac* tmp = (bls_jac*)malloc(sizeof(bls_jac) * n);
    for (size_t i = 0; i < n; i++) { bls_add_mixed(&acc, &g, &BLS_FQ); tmp[i] = acc; }
    #pragma omp parallel for num_threads(max_threads())
    for (size_t i = 0; i < n; i++) bls_to_affine(&o[i], &tmp[i], &BLS_FQ);
    free(tmp);
  } else {
    bn_aff g; memcpy(&g, g_xy, sizeof(g)); bn_jac acc; bn_jac_set_inf(&acc); bn_aff* o = (bn_aff*)out;
    bn_jac* tmp = (bn_jac*)malloc(sizeof(bn_jac) * n);
    for (size_t i = 0; i < n; i++) { bn_add_mixed(&acc, &g, &BN_FQ); tmp[i] = acc; }
    #pragma omp parallel for num_threads(max_threads())
    for (size_t i = 0; i < n; i++) bn_to_affine(&o[i], &tmp[i], &BN_FQ);
    free(tmp);
  }
  return 0;
}

int cport_fft(int curve, u64* data, unsigned log_n, int inverse, int threads) {
  init_all();
  if (threads <= 0) threads = max_threads();
  if (curve == 0) fr_fft((f4_t*)data, (int)log_n, inverse, &BLS_FR, BLS_FR_GEN, BLS_FR_S, threads);
  else fr_fft((f4_t*)data, (int)log_n, inverse, &BN_FR, BN_FR_GEN, BN_FR_S, threads);
  return 0;
}

/* ark-poly `coset_fft` / `coset_ifft` over the coset g H, g the field's multiplicative generator:
 * forward data[i] *= g^i then the FFT; inverse the inverse FFT then data[i] *= g^-i. */
static void fr_coset_scale(f4_t* a, size_t n, u64 gen, int inverse, const f4_ctx* c, int threads) {
  f4_t g = {{gen, 0, 0, 0}}; f4_to_mont(&g, &g, c);
  if (inverse) f4_inv(&g, &g, c);
  #pragma omp parallel num_threads(threads)
  {
    int nt = 1, id = 0;
#ifdef _OPENMP
    nt = omp_get_num_threads(); id = omp_get_thread_num();
#endif
    size_t lo = n * id / nt, hi = n * (id + 1) / nt;
    if (lo < hi) {
      u64 e[1] = {lo}; f4_t cur; f4_pow(&cur, &g, e, 1, c);
      for (size_t i = lo; i < hi; i++) { f4_mul(&a[i], &a[i], &cur, c); f4_mul(&cur, &cur, &g, c); }
    }
  }
}
int cport_coset_fft(int curve, u64* data, unsigned log_n, int inverse, int threads) {
  init_all();
  if (threads <= 0) threads = max_threads();
  const f4_ctx* c = curve == 0 ? &BLS_FR : &BN_FR;
  const u64 gen = curve == 0 ? BLS_FR_GEN : BN_FR_GEN;
  const int s = curve == 0 ? BLS_FR_S : BN_FR_S;
  size_t n = (size_t)1 << log_n;
  if (!inverse) fr_coset_scale((f4_t*)data, n, gen, 0, c, threads);
  fr_fft((f4_t*)data, (int)log_n, inverse, c, gen, s, threads);
  if (inverse) fr_coset_scale((f4_t*)data, n, gen, 1, c, threads);
  return 0;
}

int cport_max_threads(void) { return max_threads(); }
