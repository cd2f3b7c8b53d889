/* b2m.h -- C ABI of the H100-native (sm_90a) Marlin prover hot path.
 *
 * The reference (arkworks-rs/marlin) has no FFI; its seam is the generic parameter
 * `PC: PolynomialCommitment<F, DensePolynomial<F>>` of `Marlin<F, PC, FS>`
 * (reference src/lib.rs:64-71) and, one level down, the two upstream free functions every
 * commit/open and every AHP round bottoms out in.  Each entry point below names the
 * reference interface it replaces.  A Rust shim binding these (see INTEGRATION.md) turns the
 * library into a drop-in `PC` / prover backend.
 *
 * Conventions
 *   - Field elements cross the boundary exactly as ark-ff 0.3 stores them: little-endian
 *     u64 limbs in MONTGOMERY form (Fr: 4 limbs; Fq: 6 limbs for BLS12-381, 4 for BN254),
 *     except MSM scalars, which are canonical integers (`into_repr()`), as in
 *     `VariableBaseMSM::multi_scalar_mul(&[G::Affine], &[BigInt])`.
 *   - A G1 affine point is x||y (2*LQ u64 limbs, Montgomery); the point at infinity is
 *     encoded as x = y = 0 (never a curve point since b != 0).
 *   - Every function returns B2M_OK or an error code; b2m_last_error() gives the message.
 *     The library never aborts the host process and never falls back to the CPU.
 *   - A b2m_ctx owns one device and one stream; it is not thread-safe, distinct contexts
 *     are independent.  All calls are synchronous at return.
 */
#ifndef B2M_H
#define B2M_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum {
  B2M_OK = 0,
  B2M_ERR_INVALID_ARG = 1,
  B2M_ERR_INDEX_TOO_LARGE = 2,          /* reference src/error.rs:7  Error::IndexTooLarge */
  B2M_ERR_INSTANCE_MISMATCH = 3,        /* reference src/ahp/mod.rs:276 InstanceDoesNotMatchIndex */
  B2M_ERR_INVALID_PUBLIC_INPUT_LEN = 4, /* reference src/ahp/mod.rs:274 InvalidPublicInputLength */
  B2M_ERR_NON_SQUARE = 5,               /* reference src/ahp/mod.rs:278 NonSquareMatrix */
  B2M_ERR_DEGREE_TOO_LARGE = 6,         /* SynthesisError::PolynomialDegreeTooLarge / PC degree errors */
  B2M_ERR_MISSING_RNG = 7,              /* [U ark-poly-commit Error::MissingRng] */
  B2M_ERR_CUDA = 8,
  B2M_ERR_NCCL = 9,
  B2M_ERR_UNSUPPORTED = 10,
  B2M_ERR_SERIALIZATION = 11,           /* [U ark-serialize SerializationError::InvalidData]: an invalid point in a byte stream */
  B2M_ERR_MEMORY_LIMIT = 12             /* the byte model of a key or an index exceeds the device-memory budget (b2m_ctx_set_memory_limit) */
};

enum { B2M_CURVE_BLS12_381 = 0, B2M_CURVE_BN254 = 1, B2M_CURVE_BLS12_377 = 2 };
enum { B2M_PC_MARLIN_KZG10 = 0, B2M_PC_SONIC_KZG10 = 1 };
/* stream ciphers behind `RngCore`: rand 0.8 StdRng (= ChaCha12, `ark_std::test_rng`) and
 * rand_chacha::ChaChaRng (= ChaCha20). */
enum { B2M_RNG_CHACHA12 = 12, B2M_RNG_CHACHA20 = 20, B2M_RNG_CHACHA8 = 8,
       /* any other `RngCore`: the library pulls every random u64 through a host callback (b2m_rng::next_u64) */
       B2M_RNG_CALLBACK = 1 };

typedef struct b2m_ctx b2m_ctx;
typedef struct b2m_srs b2m_srs;
typedef struct b2m_ck b2m_ck;
typedef struct b2m_index b2m_index;

const char* b2m_last_error(void);
const char* b2m_version(void);

/* One context per GPU. */
int b2m_ctx_create(int device, b2m_ctx** out);
void b2m_ctx_destroy(b2m_ctx* ctx);
/* Number of kernel launches issued through this context so far. */
unsigned long long b2m_ctx_launches(const b2m_ctx* ctx);
/* Device-memory budget for what the library allocates: an SRS created through this context afterwards plans its layout for
 * min(free device memory, bytes) (0 = no limit: free device memory), and `index` refuses a circuit whose modelled index,
 * prover and MSM scratch exceed what the limit leaves (B2M_ERR_MEMORY_LIMIT, before anything is allocated).  The library
 * allocates from the device's default stream-ordered memory pool, which every context on that device in the process shares:
 * the limit counts the bytes the pool already holds in use, whichever context allocated them. */
int b2m_ctx_set_memory_limit(b2m_ctx* ctx, size_t bytes);
/* The device's default memory pool (shared by every context on the device in the process): out[0] = bytes in use,
 * out[1] = their high-water mark since the previous b2m_ctx_memory call on any context of that device (or since the
 * process started), out[2] = bytes the pool holds from the device.  Synchronises the context's stream and restarts the
 * high-water mark for every context of the device. */
int b2m_ctx_memory(b2m_ctx* ctx, size_t* out);
/* Multi-GPU MSM (one process per GPU of one node): rank 0 obtains an NCCL unique id (128 bytes), the
 * caller broadcasts it, every rank attaches its context.  From then on every MSM issued through the
 * context is sharded by (base, scalar) chunk across the ranks and the partial sums are exchanged with one
 * all-gather; all ranks must issue the same sequence of calls. */
int b2m_comm_unique_id(uint8_t* id, size_t cap);
int b2m_ctx_attach_comm(b2m_ctx* ctx, const uint8_t* id, size_t id_len, int rank, int world);

/* Per-kernel device timing (CUDA events on the context's stream) for the dominant kernels: enable,
 * run, then read {"kernel": {"launches", "ms", "units"}} -- units are (base, scalar) pairs for the MSM
 * kernels and points for the NTT.  Reading the report clears it. */
int b2m_ctx_profile(b2m_ctx* ctx, int enable);
int b2m_ctx_profile_report(b2m_ctx* ctx, char* json, size_t cap);

/* ---- Level 0: kernel ABI ------------------------------------------------------------- */

/* Replaces `Radix2EvaluationDomain::{fft,ifft,coset_fft,coset_ifft}_in_place(&mut Vec<F>)`
 * [U ark-poly 0.3 domain/radix2]; call sites reference src/ahp/prover.rs:321-326,350-353,
 * 359,365,427,467,488,532-545,655,681,685.  `data` is a HOST buffer of 2^log_n Fr elements
 * (natural order in and out); inverse != 0 also scales by n^-1; coset != 0 uses the coset
 * g*H with g = F::multiplicative_generator(). */
int b2m_ntt(b2m_ctx* ctx, int curve, uint64_t* data, unsigned log_n, int inverse, int coset);

/* Replaces `VariableBaseMSM::multi_scalar_mul(bases, scalars)` [U ark-ec 0.3 msm/variable_base.rs].
 * One-shot form: uploads `bases`, builds the window tables, runs the MSM, frees everything.
 * out_xy receives the affine result (Montgomery), *out_is_inf is set for the identity. */
int b2m_msm_g1(b2m_ctx* ctx, int curve, const uint64_t* bases_xy, const uint64_t* scalars, size_t n,
               uint64_t* out_xy, int* out_is_inf);

/* Device-resident committer key: the G1 powers of `PC::UniversalParams` (what `PC::trim`,
 * reference src/lib.rs:115-121, slices).  powers_of_g: n_g affine points (beta^i G);
 * powers_of_gamma_g: n_gamma affine points beta^(gamma_indices[k]) gamma G used for hiding
 * (`UniversalParams::powers_of_gamma_g` is a BTreeMap<usize, G1Affine> upstream; Marlin's PC needs
 * indices 0..=2, Sonic's additionally max_degree - bound + 0..=2 per enforced bound);
 * gamma_indices == NULL means 0..n_gamma-1.  window_bits = 0 picks the window from n_g.  The library precomputes 2^(c*w) multiples of
 * every power (HBM for doublings) so every later MSM over any contiguous slice is one
 * bucket pass. */
int b2m_srs_create(b2m_ctx* ctx, int curve, const uint64_t* powers_of_g, size_t n_g,
                   const uint64_t* powers_of_gamma_g, const uint64_t* gamma_indices, size_t n_gamma,
                   int window_bits, b2m_srs** out);
/* b2m_srs_create with a chosen number of window tables.  window_tables = 0 (what b2m_srs_create passes) keeps all
 * W = ceil(256 / c) tables whenever the byte model of the largest circuit the key can index fits the context's budget
 * (b2m_ctx_set_memory_limit), and otherwise keeps the largest T < W (at c <= 16 unless window_bits is set), and caps the
 * pairs of one MSM bucket pass, that fit; window_tables > 0 forces T (normalised to ceil(W / m) with m = ceil(W / T), the
 * tables the m bucket sets read; B2M_ERR_INVALID_ARG when m sets of 2^(c-1) buckets exceed 2^24 bucket ids).  Results do not
 * depend on the layout.  Fails with
 * B2M_ERR_MEMORY_LIMIT, naming the bytes needed and the budget, when even one table and the smallest pass do not fit, and
 * with B2M_ERR_UNSUPPORTED for T < W on a multi-GPU context. */
int b2m_srs_create_layout(b2m_ctx* ctx, int curve, const uint64_t* powers_of_g, size_t n_g,
                          const uint64_t* powers_of_gamma_g, const uint64_t* gamma_indices, size_t n_gamma,
                          int window_bits, int window_tables, b2m_srs** out);
void b2m_srs_destroy(b2m_srs* srs);
size_t b2m_srs_size(const b2m_srs* srs);
int b2m_srs_window_bits(const b2m_srs* srs);
/* Window tables the key keeps (T <= W).  Diagnostic, like b2m_srs_window_bits. */
int b2m_srs_window_tables(const b2m_srs* srs);
/* The key's layout and the byte model behind it: out[0] = window bits, [1] = window tables, [2] = pairs per MSM pass
 * (0: no cap), [3..6] = modelled bytes of the tables, the index and prover of the largest circuit, the MSM scratch, and
 * their total (with room for the pool's allocation granularity), [7] = the budget the layout was planned for (0 on a multi-GPU context, which does not plan). */
int b2m_srs_layout(const b2m_srs* srs, size_t* out);
/* Batched-affine levels the MSMs of this key run before the XYZZ bucket pass (0: none; MSMs with few bucket
 * references skip them regardless).  Diagnostic, like b2m_srs_window_bits. */
int b2m_srs_affine_levels(const b2m_srs* srs);
/* MSM over the slice powers_of_g[base_off .. base_off+n) with canonical host scalars. */
int b2m_srs_msm(b2m_srs* srs, size_t base_off, const uint64_t* scalars, size_t n, uint64_t* out_xy,
                int* out_is_inf);
/* SRS generation, the G1 half of `KZG10::setup` (reference src/lib.rs:79-96 -> [U ark-poly-commit kzg10::setup]):
 * b2m_g1_powers fills powers_of_g[i] = beta^i * g for i < n; b2m_fixed_base_msm is the general
 * `FixedBaseMSM::multi_scalar_mul(.., g, scalars)` [U ark-ec msm/fixed_base.rs] (out[i] = scalars[i] * g, e.g. the
 * powers_of_gamma_g at arbitrary exponents).  Both: one 8-bit window table of g, <= 32 mixed additions per scalar, batch
 * normalisation to affine.  beta and scalars are canonical Fr. */
int b2m_g1_powers(b2m_ctx* ctx, int curve, const uint64_t* g_xy, const uint64_t* beta, size_t n,
                  uint64_t* out_powers_xy);
int b2m_fixed_base_msm(b2m_ctx* ctx, int curve, const uint64_t* g_xy, const uint64_t* scalars, size_t n,
                       uint64_t* out_xy);

/* G2 half of `KZG10::setup` [U ark-poly-commit kzg10::setup: h, beta_h, neg_powers_of_h]: out[i] = scalars[i] * h, written as
 * ark-serialize `serialize_uncompressed` bytes (4 * sizeof(Fq) per point, infinity flag in the last byte).  h_uncompressed:
 * the G2 base in the same byte form, or NULL for the curve's standard G2 generator.  Host-side (the prover never touches G2;
 * a key needs 2 + #degree-bounds of these), no b2m_ctx needed. */
int b2m_g2_scalar_muls(int curve, const uint8_t* h_uncompressed, const uint64_t* scalars, size_t n, uint8_t* out);

/* G1 points between the device and ark-serialize files: powers_of_g[first .. first + n) of a resident SRS as
 * `serialize_uncompressed` bytes (2 * sizeof(Fq) per point: canonical little-endian x || y, infinity flag = bit 6 of the last
 * byte), and the inverse conversion of such bytes to the affine Montgomery limbs b2m_srs_create takes (no curve / subgroup
 * check: like `deserialize_unchecked`).  Conversions run on the GPU. */
int b2m_srs_export_g1(b2m_srs* srs, size_t first, size_t n, uint8_t* out);
int b2m_g1_from_uncompressed(b2m_ctx* ctx, int curve, const uint8_t* bytes, size_t n, uint64_t* out_xy);
int b2m_g1_to_uncompressed(b2m_ctx* ctx, int curve, const uint64_t* points_xy, size_t n, uint8_t* out);

/* Checked decoding of ark-serialize points, `CanonicalDeserialize::deserialize` (compressed != 0) or
 * `deserialize_uncompressed` semantics [U ark-serialize / ark-ec 0.3]: the flag bits (both set is invalid), every coordinate
 * below p, the curve equation (compressed: a square root exists, and the sign bit picks the root) and the prime-order
 * subgroup (BLS12-381 G1 by the endomorphism test phi(P) = -u^2 P; G2 by r * Q = O; BN254 G1 has cofactor 1).  Runs on the
 * GPU, one thread per point, in chunks of 2^18 points, so device memory stays bounded whatever n is.
 *   G1: bytes = n * sizeof(Fq) (compressed) or n * 2 sizeof(Fq); out_xy = n affine Montgomery points (infinity = 0, 0).
 *   G2: bytes = n * 2 sizeof(Fq) or n * 4 sizeof(Fq) (x = c0 || c1, flags in the top of the last byte); out_uncompressed =
 *       n * 4 sizeof(Fq) canonical bytes, the form b2m_g2_scalar_muls writes and b2m_vk_create takes.
 * An invalid point fails with B2M_ERR_SERIALIZATION; *bad_index receives the lowest invalid index and *bad_reason its cause
 * (1 both flags set, 2 x >= p, 3 not on the curve, 4 not in the subgroup, 5 y >= p), and b2m_last_error() names both; the
 * output is then incomplete.  On success *bad_index = n and *bad_reason = 0.  bad_index / bad_reason may be NULL. */
int b2m_g1_decode_ark(b2m_ctx* ctx, int curve, const uint8_t* bytes, size_t n, int compressed, uint64_t* out_xy,
                      size_t* bad_index, int* bad_reason);
int b2m_g2_decode_ark(b2m_ctx* ctx, int curve, const uint8_t* bytes, size_t n, int compressed, uint8_t* out_uncompressed,
                      size_t* bad_index, int* bad_reason);
/* Checked decoding of snarkjs "LEM" points, the form of a Powers-of-Tau (.ptau) file: uncompressed, every Fq (every Fq2 component,
 * c0 then c1) little-endian Montgomery limbs with R = 2^(64 * limbs), no flags, all-zero bytes = infinity.  Same checks,
 * chunking and status contract as b2m_g1_decode_ark / b2m_g2_decode_ark: each coordinate limb vector < p (a non-reduced
 * representative is invalid: 2 x, 5 y), the curve equation (3) and the prime-order subgroup (4).  Infinity decodes with status
 * OK; callers that need a finite point check for it.  Any curve id is accepted.
 *   G1: bytes = n * 2 sizeof(Fq); out_xy = n affine Montgomery points (infinity = 0, 0).
 *   G2: bytes = n * 4 sizeof(Fq); out_uncompressed = n * 4 sizeof(Fq) canonical ark bytes (the b2m_vk_create form). */
int b2m_g1_decode_lem(b2m_ctx* ctx, int curve, const uint8_t* bytes, size_t n, uint64_t* out_xy, size_t* bad_index, int* bad_reason);
int b2m_g2_decode_lem(b2m_ctx* ctx, int curve, const uint8_t* bytes, size_t n, uint8_t* out_uncompressed, size_t* bad_index,
                      int* bad_reason);
/* `PairingEngine::product_of_pairings(pairs).is_one()` [U ark-ec 0.3] for many products at once.  g2: n_g2 distinct G2 points
 * as uncompressed ark-serialize bytes (the b2m_g2_scalar_muls / b2m_vk_create form).  Product k is the pairs
 * [product_off[k], product_off[k+1]): G1 point g1_xy[j] (affine Montgomery, (0,0) = infinity) with G2 point g2_index[j].
 * verdicts[k] = 1 iff the product is one (an empty product is one).  A pair with either point at infinity contributes 1.
 * Runs on the GPU, one thread per product, with the optimal-ate Miller loop and final exponentiation of pairing.cuh; the G2
 * line coefficients are computed once per call on the host.  Products go to the GPU in chunks of at most 2^16 products and
 * max(2^18, pairs of the largest product) pairs, so device scratch stays bounded by that whatever n_products is.
 * Input checks: a G2 point that is non-canonical or off the twist fails with B2M_ERR_SERIALIZATION, a G1 point off the curve
 * (or with limbs not below p) with B2M_ERR_INVALID_ARG, as do decreasing offsets and g2_index[j] >= n_g2; b2m_last_error()
 * names the index.  Subgroup membership is the caller's job: b2m_g1_decode_ark / b2m_g2_decode_ark check it. */
int b2m_pairing_check(b2m_ctx* ctx, int curve, size_t n_g2, const uint8_t* g2, size_t n_products, const size_t* product_off,
                      const uint64_t* g1_xy, const uint32_t* g2_index, int* verdicts);
/* `CanonicalSerialize::serialize` (compressed) of G1 points given as affine Montgomery limbs (GPU), and of G2 points given as
 * uncompressed canonical bytes (host: no square root is needed).  Infinity is written as zero coordinates + bit 6. */
int b2m_g1_to_compressed(b2m_ctx* ctx, int curve, const uint64_t* points_xy, size_t n, uint8_t* out);
int b2m_g2_to_compressed(int curve, const uint8_t* uncompressed, size_t n, uint8_t* out);

/* Fr elements between the device and ark-serialize files (the index-key loader, marlin_b200/keyfile.py): canonical
 * little-endian bytes (32 per element) to Montgomery limbs with `deserialize` semantics -- every value must be below r --
 * and back.  Both run on the GPU, one thread per element, the decoder in chunks of 2^18 elements and the encoder in chunks
 * of 2^20 elements, so device scratch stays bounded whatever n is.  An element >= r fails with
 * B2M_ERR_SERIALIZATION and *bad_index receives the lowest such index (n on success; bad_index may be NULL). */
int b2m_fr_decode_ark(b2m_ctx* ctx, int curve, const uint8_t* bytes, size_t n, uint64_t* out_limbs, size_t* bad_index);
int b2m_fr_to_canonical(b2m_ctx* ctx, int curve, const uint64_t* limbs, size_t n, uint8_t* out);
/* `Radix2EvaluationDomain::new(2^log_size)` as ark-serialize writes it [U ark-poly 0.3 domain/radix2]: size (u64),
 * log_size_of_group (u32), then size_as_field_element, size_inv, group_gen, group_gen_inv, generator_inv as canonical Fr
 * (12 + 5 * 32 = 172 bytes).  Host-side, no b2m_ctx needed. */
int b2m_domain_ark(int curve, unsigned log_size, uint8_t* out);
/* The row lengths of an ark-serialize `Vec<Vec<T>>` with fixed-size entries (a `Matrix<F>` has entry_bytes = 40: F then
 * usize), after its outer u64 length: bytes[0 .. len) is the rest of the file.  row_ptr (n_rows + 1) receives the prefix sums
 * of the row lengths and *end the byte length of the n_rows rows.  A row whose length field is cut short (bad_reason 1) or
 * whose entries run past len (bad_reason 2) fails with B2M_ERR_SERIALIZATION, *bad_row = its index, *end = the offset of its
 * length field.  Host-side, no b2m_ctx needed. */
int b2m_ark_matrix_rows(const uint8_t* bytes, size_t len, size_t n_rows, size_t entry_bytes, uint64_t* row_ptr, size_t* end,
                        size_t* bad_row, int* bad_reason);

/* circom `.r1cs` files [U circom r1csfile]: section 2 holds m constraints, each three linear combinations A, B, C, each a
 * u32 term count followed by that many (u32 wire, 32-byte canonical little-endian coefficient) terms (n8 = 32).
 *
 * b2m_circom_constraint_rows walks the term counts once on the host (no context) and writes the three term-count prefix
 * sums row_ptr_{a,b,c}[0..=m].  LC j of constraint k then starts at byte 4 (3k + j) + 36 (terms before it).  *end receives
 * the bytes the m constraints take (a caller compares it with the section size).  A count truncated by len
 * (*bad_reason = 1) or terms running past len (2) fail with B2M_ERR_SERIALIZATION; *bad_constraint receives the
 * constraint and b2m_last_error() names it and its matrix, e.g. "constraints[12].B: truncated in the term count".
 *
 * b2m_circom_decode_constraints decodes the section on the GPU, in chunks of whole constraints (device scratch stays
 * bounded): wire w goes to column w when w < ni0 (= 1 + nPubOut + nPubIn) and to w + shift otherwise (the instance padding
 * of Marlin's indexer), coefficients to Montgomery form, and every row to normal form: columns ascending, equal columns
 * summed mod r, zero sums dropped.  out_row_ptr[j] receives m + 1 entries; out_col[j] / out_coeff[j] (4 u64 limbs each)
 * must hold row_ptrs[j][m] entries, as normalising never adds one; matrix j ends with out_row_ptr[j][m] entries.  A wire
 * >= n_wires (*bad_reason = 1) or a coefficient not below r (2) fails with B2M_ERR_SERIALIZATION; *bad_matrix (0/1/2 =
 * A/B/C) and *bad_term (index into that matrix's terms, row_ptrs[j]) name the lowest such term in file order.
 *
 * b2m_r1cs_check is ark-relations' `which_is_unsatisfied` for any padded R1CS (the b2m_index_create form, with the
 * formatted instance and the witness as b2m_prove takes them): *bad_row receives the lowest row r with
 * <A_r, z> * <B_r, z> != <C_r, z>, or nc when every row holds.  A column >= nv fails with B2M_ERR_INVALID_ARG.  The prover
 * does not call it: as in the reference, proving an unsatisfied instance is not refused. */
int b2m_circom_constraint_rows(const uint8_t* bytes, size_t len, size_t m, uint64_t* row_ptr_a, uint64_t* row_ptr_b, uint64_t* row_ptr_c,
                               size_t* end, size_t* bad_constraint, int* bad_reason);
int b2m_circom_decode_constraints(b2m_ctx* ctx, int curve, const uint8_t* bytes, size_t len, size_t m, const uint64_t* const* row_ptrs,
                                  uint64_t n_wires, uint64_t ni0, uint64_t shift, uint64_t* const* out_row_ptr, uint64_t* const* out_col,
                                  uint64_t* const* out_coeff, int* bad_matrix, size_t* bad_term, int* bad_reason);

/* The caller's `zk_rng: &mut R` / `rng: Option<&mut dyn RngCore>` (reference src/lib.rs:154,125).  Two forms:
 *  - kind = B2M_RNG_CHACHA8/12/20, the fast path for the generators the reference's tests and benches use
 *    (`ark_std::test_rng()` = ChaCha12, `rand_chacha::ChaChaRng` = ChaCha20): the stream is described by its key and
 *    word position, so the mask polynomial (3|H| draws, src/ahp/prover.rs:371) is sampled on the device bit-exactly;
 *    word_pos is updated to the position after the call.
 *  - kind = B2M_RNG_CALLBACK, any other generator: every `next_u64()` the reference would issue is pulled, in the
 *    reference's order, through `next_u64(state)` on the calling thread (a Rust shim passes a trampoline over
 *    `&mut dyn RngCore`); the mask polynomial is then drawn on the host and uploaded once.  key / word_pos are unused.
 * Draw order and counts are those of ark-ff 0.3 `F::rand` (4 u64 limbs per attempt, low limb first, rejection sampling). */
typedef struct {
  int kind;          /* B2M_RNG_CHACHA* or B2M_RNG_CALLBACK */
  uint8_t key[32];
  uint64_t word_pos; /* number of 32-bit words already consumed from the stream */
  uint64_t (*next_u64)(void* state); /* B2M_RNG_CALLBACK only */
  void* state;
} b2m_rng;

/* Is the key one chain of powers?  With P_i = powers_of_g[i] (D = b2m_srs_size - 1), G_k the gamma power of key k held on the
 * device and N_k = neg_h[j] for key k = neg_keys[j] (optional: SonicKZG10's beta^-k h), decides all of
 *   (0) e(P_{i+1}, h) = e(P_i, beta_h)  for i < D          (1) e(G_{k+1}, h) = e(G_k, beta_h)  for held keys k, k + 1
 *   (2) e(P_k, N_k)   = e(P_0, h)       for every neg key  (3) e(G_k, N_k)   = e(G_0, h)       for every neg key with G_k held
 * h, beta_h and neg_h are uncompressed ark G2 bytes (b2m_g2_decode_ark / _lem output; their subgroup is the caller's check).
 * One randomised check on the GPU -- two D-pair MSMs over the window tables, a few one-pair MSMs, one pairing product of
 * 3 + n_neg pairs -- and, when it fails, bisection with fresh randomisers.  *ok = 1 when every relation holds; otherwise *ok = 0,
 * *bad_kind = the family (0-3) and *bad_index = i (family 0) or the key k of the lowest failing relation of the first failing
 * family.  A bad relation passes a check with probability at most 2^-128.  Randomisers: two next_u64() per relation and check,
 * family 0 in ascending i (ChaCha: generated on the device at the stream position, which is advanced), then families 1-3.
 * Errors: B2M_ERR_MISSING_RNG without a usable rng, B2M_ERR_UNSUPPORTED on a multi-GPU context, B2M_ERR_INVALID_ARG for h /
 * beta_h / neg_h at infinity or a neg key above D, B2M_ERR_SERIALIZATION for a G2 point off the twist. */
int b2m_srs_check_powers(b2m_srs* srs, const uint8_t* h, const uint8_t* beta_h, size_t n_neg, const uint64_t* neg_keys,
                         const uint8_t* neg_h, b2m_rng* rng, int* ok, int* bad_kind, size_t* bad_index);

/* ---- Level 1: polynomial-commitment ABI --------------------------------------------------------- */

/* Replaces `PC::commit(ck, polynomials, rng)` for PC = MarlinKZG10 / SonicKZG10 [U ark-poly-commit 0.3
 * marlin_pc/mod.rs, sonic_pc/mod.rs commit -> kzg10::KZG10::commit]; call sites reference
 * src/lib.rs:125,172,193,213.  Polynomials are host coefficient arrays (Montgomery Fr, low degree first)
 * committed in order with the blinding polynomials drawn from `rng` exactly as the reference does
 * (hiding_bound h draws h + 2 coefficients; MarlinKZG10 draws a second set for the shifted commitment).
 *   degree_bounds[i] / hiding_bounds[i] : -1 for None.
 *   out_comm_xy[i]      affine commitment; out_shifted_xy[i]: MarlinKZG10 shifted commitment of a bounded
 *                        polynomial (all-zero when absent; unused for SonicKZG10).
 *   out_rand / out_shifted_rand : blinding polynomial coefficients, rand_stride Fr per polynomial (zero padded).
 * rng may be NULL when no polynomial is hiding (B2M_ERR_MISSING_RNG otherwise). */
int b2m_pc_commit(b2m_srs* srs, int pc_variant, size_t n_polys, const uint64_t* const* coeffs,
                  const size_t* n_coeffs, const int64_t* degree_bounds, const int64_t* hiding_bounds,
                  b2m_rng* rng, uint64_t* out_comm_xy, uint64_t* out_shifted_xy, uint64_t* out_rand,
                  uint64_t* out_shifted_rand, size_t rand_stride);

/* Replaces `PC::open_individual_opening_challenges(ck, polynomials, commitments, point, challenges, rands)`
 * for one point [U ark-poly-commit 0.3 marlin_pc/mod.rs, sonic_pc/mod.rs -> kzg10::KZG10::open], the call the
 * generic `open_combinations` / `batch_open` code ends in (reference src/lib.rs:292-302).  Polynomials and their
 * commitment randomness are given in query order; challenge k is opening_challenge^k starting at k = 0
 * (MarlinKZG10 spends a second challenge on every degree-bounded polynomial).  max_degree_bound: the largest
 * enforced bound of the committer key (MarlinKZG10 shifted powers), -1 if none.
 * Output: the `kzg10::Proof { w, random_v }`. */
int b2m_pc_open(b2m_srs* srs, int pc_variant, size_t n_polys, const uint64_t* const* coeffs,
                const size_t* n_coeffs, const int64_t* degree_bounds, const uint64_t* rands,
                const uint64_t* shifted_rands, size_t rand_stride, int64_t max_degree_bound,
                const uint64_t* point, const uint64_t* opening_challenge, uint64_t* out_w_xy,
                int* out_has_random_v, uint64_t* out_random_v);

/* Replaces `PC::trim(pp, supported_degree, supported_hiding_bound, enforced_degree_bounds)` (reference src/lib.rs:112-121)
 * for PC = MarlinKZG10 / SonicKZG10 [U ark-poly-commit 0.3 marlin_pc/mod.rs, sonic_pc/mod.rs trim].  The device-resident
 * SRS already holds every power, so trimming selects and validates: supported_degree <= max_degree, the hiding bound needs
 * powers 0..=supported_hiding_bound+1 of gamma*G (SonicKZG10 additionally max_degree - bound + 0..=hiding_bound+1 per enforced
 * bound), every enforced bound <= supported_degree.  The committer key borrows the SRS (destroy the key first).
 * Errors: B2M_ERR_DEGREE_TOO_LARGE (TrimmingDegreeTooLarge / bound above the supported degree), B2M_ERR_INVALID_ARG. */
int b2m_trim(b2m_srs* srs, int pc_variant, size_t supported_degree, size_t supported_hiding_bound,
             const uint64_t* enforced_degree_bounds, size_t n_bounds, b2m_ck** out);
void b2m_ck_destroy(b2m_ck* ck);
size_t b2m_ck_supported_degree(const b2m_ck* ck);
/* `vk.degree_bounds_and_shift_powers` of MarlinKZG10's verifier key: shift power for an enforced bound =
 * powers_of_g[max_degree - bound] (affine x||y Montgomery).  B2M_ERR_INVALID_ARG if the bound is not enforced. */
int b2m_ck_shift_power(const b2m_ck* ck, uint64_t bound, uint64_t* out_xy);
/* `PC::commit(ck, ..)` with the committer key's checks [U ark-poly-commit check_degrees_and_bounds]: a polynomial longer than
 * supported_degree + 1 coefficients, a degree bound that is not one of the enforced bounds (or below the polynomial's degree)
 * or a hiding bound above the supported one fail with B2M_ERR_DEGREE_TOO_LARGE / B2M_ERR_INVALID_ARG.  Otherwise identical
 * to b2m_pc_commit. */
int b2m_ck_commit(b2m_ck* ck, size_t n_polys, const uint64_t* const* coeffs, const size_t* n_coeffs,
                  const int64_t* degree_bounds, const int64_t* hiding_bounds, b2m_rng* rng, uint64_t* out_comm_xy,
                  uint64_t* out_shifted_xy, uint64_t* out_rand, uint64_t* out_shifted_rand, size_t rand_stride);

/* Replaces `PC::open_combinations(ck, lc_s, polynomials, commitments, query_set, opening_challenge, rands, rng)`
 * (reference src/lib.rs:292-302) [U ark-poly-commit 0.3 marlin_pc / sonic_pc open_combinations_individual_opening_challenges].
 *   polynomials / rands       : as for b2m_pc_commit / b2m_pc_open (hiding[i] != 0 iff polynomial i was committed hiding).
 *   linear combinations       : LC l has the terms [lc_term_off[l], lc_term_off[l+1]); term t is lc_coeff[t] (Montgomery Fr)
 *                               times polynomial lc_poly[t], or the constant `LCTerm::One` when lc_poly[t] < 0 (which only
 *                               shifts the evaluation and is skipped, as upstream does).  The caller passes the LCs in the
 *                               order of their labels (upstream sorts them, reference src/ahp/mod.rs:219).  An LC may carry a
 *                               degree bound only if it is a single polynomial with coefficient one
 *                               (else B2M_ERR_INVALID_ARG: EquationHasDegreeBounds).
 *   query set                 : pairs (query_lc[q], query_point[q]); points[] are the distinct evaluation points in the order
 *                               of their point labels (upstream iterates a BTreeMap keyed by the label: "beta" < "gamma").
 *   opening challenge         : xi; challenge k is xi^k, restarting at k = 0 for every point.
 * Output: one `kzg10::Proof {w, random_v}` per point -- `BatchLCProof.proof` (its `evals` field is None upstream). */
int b2m_ck_open_combinations(b2m_ck* ck, size_t n_polys, const uint64_t* const* coeffs, const size_t* n_coeffs,
                             const int64_t* degree_bounds, const int* hiding, const uint64_t* rands,
                             const uint64_t* shifted_rands, size_t rand_stride, size_t n_lcs, const size_t* lc_term_off,
                             const int64_t* lc_poly, const uint64_t* lc_coeff, size_t n_queries, const size_t* query_lc,
                             const size_t* query_point, size_t n_points, const uint64_t* points,
                             const uint64_t* opening_challenge, uint64_t* out_w_xy, int* out_has_random_v,
                             uint64_t* out_random_v);

/* `PC::VerifierKey` of MarlinKZG10 / SonicKZG10 [U ark-poly-commit 0.3 marlin_pc / sonic_pc VerifierKey], the key of
 * b2m_pc_check_combinations, built from public data.  The key borrows the context, like b2m_vk.
 *   max_degree           : the SRS max degree D (every bound must be <= D)
 *   g_xy, gamma_g_xy     : powers_of_g[0] and powers_of_gamma_g[0] (affine x||y Montgomery)
 *   h_bytes, beta_h_bytes: uncompressed G2 bytes, checked to be finite points of the twist (as b2m_vk_create checks them)
 *   bounds[n_bounds]     : the enforced degree bounds (distinct)
 *   bound_points         : per bound, MarlinKZG10: `degree_bounds_and_shift_powers`, the G1 point powers_of_g[D - bound] (x||y
 *                          Montgomery limbs); SonicKZG10: `degree_bounds_and_neg_powers_of_h`, beta^-(D - bound) h (uncompressed G2)
 * Errors: B2M_ERR_INVALID_ARG. */
typedef struct b2m_pc_vk b2m_pc_vk;
int b2m_pc_vk_create(b2m_ctx* ctx, int curve, int pc_variant, size_t max_degree, const uint64_t* g_xy, const uint64_t* gamma_g_xy,
                     const uint8_t* h_bytes, const uint8_t* beta_h_bytes, size_t n_bounds, const uint64_t* bounds,
                     const void* bound_points, b2m_pc_vk** out);
void b2m_pc_vk_destroy(b2m_pc_vk* vk);

/* `PC::check_combinations(vk, lc_s, commitments, query_set, evaluations, proof, opening_challenge, rng)` [U ark-poly-commit 0.3
 * marlin_pc / sonic_pc check_combinations_individual_opening_challenges] for n_sets independent sets in one call.  `batch_check`
 * is the case where every LC is one commitment with coefficient one, labelled as the commitment, and `check` is `batch_check` at
 * one point: callers form those LCs themselves.  Set s owns consecutive ranges of the arrays below; every index inside a set
 * (commitment, LC, point) is local to the set.  What the prover sends is ark-serialize bytes, what the verifier forms is
 * Montgomery Fr limbs (4 u64):
 *   commitments   : [comm_off[s], comm_off[s+1]): comms (compressed G1, sizeof(Fq) bytes each), comm_bounds (degree bound, -1 for
 *                   None), and for MarlinKZG10 has_shifted / shifted (the compressed `shifted_comm`, read where has_shifted != 0 and
 *                   the commitment is bounded; both may be NULL for SonicKZG10)
 *   LCs           : [lc_off[s], lc_off[s+1]), in label order; LC l (a global index) has the terms [lc_term_off[l], lc_term_off[l+1]):
 *                   lc_coeff[t] (Montgomery) times commitment lc_comm[t], or `LCTerm::One` when lc_comm[t] = -1
 *   opening points: [point_off[s], point_off[s+1]), distinct, in point-label order: points (Montgomery), and the point's
 *                   `kzg10::Proof` -- w (compressed G1), has_random_v, random_v (32 canonical little-endian bytes)
 *   queries       : [query_off[s], query_off[s+1]): (query_lc, query_point) and the evaluation evals (32 canonical bytes)
 *   challenges    : xi per set (Montgomery); challenge k is xi^k over the point's LCs in label order, MarlinKZG10 spending a
 *                   second one on each degree-bounded LC
 * verdicts[s] = 1 accepted, 0 rejected by the check, -1 malformed: a point that does not decode (b2m_g1_decode_ark's checks:
 * flags, x < p, curve, BLS12-381 subgroup), an evaluation or random_v not below r, a bounded MarlinKZG10 commitment without
 * has_shifted.  The points are decoded on the GPU; the checks of all sets are folded with one 128-bit randomiser per (set,
 * point) from rng into a few MSMs and one pairing product on the GPU, and a failing batch is bisected with fresh randomisers
 * as b2m_verify_batch does (DESIGN.md §16).  Upstream's `Err` cases fail the call with B2M_ERR_INVALID_ARG naming the set,
 * before any work or rng draw: a bounded commitment in an LC of several terms (EquationHasDegreeBounds) or with a coefficient
 * other than one, a degree bound the key does not enforce, an index out of its set's range, a repeated query, a point without
 * a query.  rng == NULL fails with B2M_ERR_MISSING_RNG.  n_sets = 0 is allowed. */
int b2m_pc_check_combinations(b2m_pc_vk* vk, size_t n_sets, const size_t* comm_off, const uint8_t* comms, const int64_t* comm_bounds,
                              const int* has_shifted, const uint8_t* shifted, const size_t* lc_off, const size_t* lc_term_off,
                              const int64_t* lc_comm, const uint64_t* lc_coeff, const size_t* point_off, const uint64_t* points,
                              const uint8_t* w, const int* has_random_v, const uint8_t* random_v, const size_t* query_off,
                              const size_t* query_lc, const size_t* query_point, const uint8_t* evals, const uint64_t* challenges,
                              b2m_rng* rng, int* verdicts);
/* Phase split of the last b2m_pc_check_combinations on this key, with b2m_verify_timings's keys where they apply: {"sets",
 * "points", "decode_ms", "terms_ms" (the equations' bookkeeping, host threads), "g2_set_ms", "msm_tables_ms", "fold_ms" (the
 * randomised scalar fold of every check, host), "msm_ms", "pairing_ms", "first_check_ms", "bisection_ms", "checks",
 * "products", "total_ms"}. */
int b2m_pc_vk_timings(const b2m_pc_vk* vk, char* json, size_t cap);

/* ---- Level 2: prover ABI ---------------------------------------------------------------- */

/* R1CS matrix in CSR form, as `ConstraintSystem::to_matrices()` yields it
 * (reference src/ahp/indexer.rs:81 `Matrix<F> = Vec<Vec<(F, usize)>>`): row r holds entries
 * [row_ptr[r], row_ptr[r+1]); coeff is Montgomery Fr (4 u64 each). */
typedef struct {
  const uint64_t* row_ptr; /* num_constraints + 1 */
  const uint64_t* col;     /* nnz column (variable) indices */
  const uint64_t* coeff;   /* nnz * 4 limbs */
} b2m_matrix;

/* (b2m_r1cs_check: see the circom section above) */
int b2m_r1cs_check(b2m_ctx* ctx, int curve, size_t nc, size_t nv, size_t ni, const b2m_matrix* a, const b2m_matrix* b, const b2m_matrix* c,
                   const uint64_t* instance, const uint64_t* witness, size_t* bad_row);

/* Replaces `Marlin::index` (reference src/lib.rs:100-148): AHP indexer
 * (src/ahp/indexer.rs:151-234, src/ahp/constraint_systems.rs:125-262) + `PC::trim` +
 * commitment to the six index polynomials.  The matrices must already be padded/squared
 * (num_constraints == num_variables) as `make_matrices_square_for_indexer` leaves them.
 * Rows need not be in column order.  num_instance_variables (the formatted input, leading one
 * included) must be a power of two (B2M_ERR_INVALID_PUBLIC_INPUT_LEN) and may equal
 * num_variables (no witness at all); a column index >= num_variables is B2M_ERR_INVALID_ARG.
 * vk_bytes receives `IndexVerifierKey::write` (ToBytes) output: index_info || index_comms. */
int b2m_index_create(b2m_srs* srs, int pc_variant, size_t num_constraints, size_t num_variables,
                     size_t num_instance_variables, const b2m_matrix* a, const b2m_matrix* b,
                     const b2m_matrix* c, b2m_index** out);
void b2m_index_destroy(b2m_index* idx);
/* Serialized `index_vk` as the transcript sees it (ToBytes, reference src/data_structures.rs:36-43). */
int b2m_index_vk_bytes(const b2m_index* idx, uint8_t* out, size_t cap, size_t* len);
/* Commitments to the index polynomials (affine x||y Montgomery, 6 points). */
int b2m_index_comms(const b2m_index* idx, uint64_t* out_xy);

/* An index from an `IndexProverKey` file instead of from `Marlin::index`: the matrices (as b2m_index_create takes them; the
 * index keeps them in this row form for b2m_index_export), num_non_zero = |joint matrix| (index_info.num_non_zero) and the
 * twelve index vectors as canonical little-endian Fr bytes in HOST memory (e.g. a memory-mapped file): vectors[0..6) the
 * coefficients of row, col, a_val, b_val, c_val, row_col (vector_lens[i] <= |K|, zero-padded to |K|), vectors[6..12) their
 * evaluations on K in the same order (vector_lens[i] == |K|).  index_comms_xy: the six commitments (affine x||y Montgomery).
 * The vectors are decoded on the GPU straight into the index's device buffers; no arithmetization and no commitment MSM
 * runs.  Checked on the GPU: every element is below r, and the NTT over K of each zero-padded coefficient vector equals its
 * evaluations.  check_commitments != 0 also recomputes the six commitments (`PC::commit`, rng = None) and compares them.
 * A failed check returns B2M_ERR_SERIALIZATION with *bad_vector (0..11, or 0..5 for a commitment), *bad_index (the lowest
 * bad element) and *bad_reason (1 not below r, 2 evaluations differ from the NTT of the coefficients, 3 commitment
 * differs); the pointers may be NULL.  Dimension errors are those of b2m_index_create, and num_non_zero must lie between
 * the entry count of the largest matrix and the sum of the three. */
int b2m_index_load(b2m_srs* srs, int pc_variant, size_t num_constraints, size_t num_variables, size_t num_instance_variables,
                   size_t num_non_zero, const b2m_matrix* a, const b2m_matrix* b, const b2m_matrix* c,
                   const uint8_t* const* vectors, const size_t* vector_lens, const uint64_t* index_comms_xy,
                   int check_commitments, size_t* bad_vector, size_t* bad_index, int* bad_reason, b2m_index** out);
/* num_non_zero, |K| and the entries of A, B, C (matrix_nnz[3]) of an index: the buffer sizes b2m_index_export needs. */
int b2m_index_sizes(const b2m_index* idx, size_t* num_non_zero, size_t* domain_k, size_t* matrix_nnz);
/* The index as an `IndexProverKey` file holds it, converted on the GPU: vectors (12 * |K| * 32 bytes) receives the
 * coefficient vectors (zero-padded to |K|) then the evaluation vectors, in b2m_index_load's order, as canonical Fr bytes;
 * row_ptrs[m] (num_constraints + 1), cols[m] (matrix_nnz[m]) and coeffs[m] (32 * matrix_nnz[m] canonical bytes) receive
 * matrix m = A, B, C in the row form the index was given.  Any output pointer may be NULL to skip it. */
int b2m_index_export(b2m_index* idx, uint8_t* vectors, uint64_t* const* row_ptrs, uint64_t* const* cols,
                     uint8_t* const* coeffs);
/* Where the index keeps its twelve |K|-vectors: *host = 0 in device memory, 1 in pinned host memory, streamed to the GPU
 * in round 3 and the opening of every proof; *host_bytes = the pinned bytes (0 when device-resident).  `index` and
 * `load_index` choose host residency only when the device-memory model of the device-resident index does not fit and the
 * host-resident one does (single-GPU contexts; environment B2M_INDEX_HOST=1 forces it, for tests).  Either pointer may be
 * NULL. */
int b2m_index_residency(const b2m_index* idx, int* host, size_t* host_bytes);


/* Replaces `Marlin::prove` (reference src/lib.rs:151-311).  formatted_input: the instance
 * assignment including the leading one (|X| elements); witness: the witness assignment
 * (num_variables - |X| elements), both Montgomery Fr.  proof receives the
 * `CanonicalSerialize` bytes of `Proof<F, PC>` (reference src/data_structures.rs:100-110). */
int b2m_prove(b2m_index* idx, const uint64_t* formatted_input, size_t n_input,
              const uint64_t* witness, size_t n_witness, b2m_rng* zk_rng, uint8_t* proof,
              size_t cap, size_t* proof_len);

/* Copy an instance into HBM ahead of time.  A later b2m_prove(idx, NULL, 0, NULL, 0, ...) proves the
 * staged instance without any host-to-device input traffic (bench.py's device-resident timing). */
int b2m_index_stage(b2m_index* idx, const uint64_t* formatted_input, size_t n_input,
                    const uint64_t* witness, size_t n_witness);

/* Per-phase device timings of the last b2m_prove on this index (milliseconds), labelled
 * with the reference's own timer names (ark_std start_timer! labels, SURVEY.md section 5). */
int b2m_prove_timings(const b2m_index* idx, char* json, size_t cap);

/* ---- Level 2: verifier ABI -------------------------------------------------------------- */

/* `IndexVerifierKey` plus the verifier half of the trimmed SRS (reference src/lib.rs:315-433 reads both), built from public
 * data only.  The key borrows the context (destroy the key first, or the context is freed with its last child).
 *   index_comms_xy : the six index commitments (row, col, a_val, b_val, c_val, row_col), affine x||y Montgomery
 *   g_xy, gamma_g_xy : powers_of_g[0] and powers_of_gamma_g[0] of the SRS
 *   h_bytes, beta_h_bytes : G2 points as ark-serialize uncompressed bytes (the b2m_g2_scalar_muls / SRS-file form),
 *                    checked to be finite points of the curve
 *   bounds[n_bounds] : the enforced degree bounds; they must include |H| - 2 and |K| - 2 of this index
 *   bound_points   : per bound, MarlinKZG10: the G1 shift power powers_of_g[D - bound] (x||y Montgomery limbs, D = the SRS
 *                    max degree); SonicKZG10: neg_powers_of_h[D - bound] = beta^-(D - bound) h (uncompressed G2 bytes)
 * Errors: B2M_ERR_NON_SQUARE (num_constraints != num_variables), B2M_ERR_INVALID_ARG. */
typedef struct b2m_vk b2m_vk;
int b2m_vk_create(b2m_ctx* ctx, int curve, int pc_variant, size_t num_constraints, size_t num_variables, size_t num_non_zero,
                  const uint64_t* index_comms_xy, const uint64_t* g_xy, const uint64_t* gamma_g_xy, const uint8_t* h_bytes,
                  const uint8_t* beta_h_bytes, size_t n_bounds, const uint64_t* bounds, const void* bound_points, b2m_vk** out);
void b2m_vk_destroy(b2m_vk* vk);

/* `Marlin::verify` (reference src/lib.rs:315-433) for n proofs under one key.  public_inputs[i]: n_inputs[i] Montgomery Fr
 * (the unformatted input, as Marlin::verify takes it); proofs[i]: proof_lens[i] `CanonicalSerialize` bytes of `Proof<F, PC>`.
 * verdicts[i] = 1 accepted, 0 rejected by the check, -1 malformed bytes (framing, trailing bytes, x >= p, a point not on the
 * curve or outside the prime-order subgroup, an evaluation or random_v >= r).  Malformed proofs are verdicts, not errors.
 * The proofs' G1 points are decoded on the GPU; all checks of the batch are folded with one 128-bit randomiser per (proof,
 * opening point) drawn from rng (which must be unpredictable to the prover) into a few MSMs and one pairing product
 * (b2m_pairing_check's kernel), all on the GPU; a failing batch is bisected with fresh randomisers until every bad proof is isolated.
 * rng == NULL fails with B2M_ERR_MISSING_RNG. */
int b2m_verify_batch(b2m_vk* vk, size_t n, const uint64_t* const* public_inputs, const size_t* n_inputs,
                     const uint8_t* const* proofs, const size_t* proof_lens, b2m_rng* rng, int* verdicts);
/* A batch of one: *ok receives the verdict (1, 0 or -1). */
int b2m_verify(b2m_vk* vk, const uint64_t* public_input, size_t n_input, const uint8_t* proof, size_t proof_len,
               b2m_rng* rng, int* ok);
/* `Marlin::verify` for n proofs under n_keys verifier keys at once.  Proof i is checked under vks[key_of[i]].  All keys must
 * belong to the same b2m_ctx and curve; PC variants and SRSs may differ, and a key may appear more than once.  Verdicts, rng
 * requirements and malformed-proof handling are those of b2m_verify_batch; verdicts[i] equals what
 * b2m_verify_batch(vks[key_of[i]], ...) gives proof i.  Keys whose SRSs share h and beta h share one G2 group: every check
 * folds all its proofs into one set of MSMs and decides one pairing product per G2 group, all products of a bisection level
 * in one launch.  Randomisers are drawn as b2m_verify_batch draws them, in item order, so one key gives exactly its draws.
 * A null key, keys of two contexts or curves and key_of[i] >= n_keys fail with B2M_ERR_INVALID_ARG naming the index, before
 * any work or rng draw; rng as b2m_verify_batch.  n = 0 is allowed.  The call's timings go to every key in vks. */
int b2m_verify_multi(size_t n_keys, b2m_vk* const* vks, size_t n, const uint32_t* key_of,
                     const uint64_t* const* public_inputs, const size_t* n_inputs, const uint8_t* const* proofs,
                     const size_t* proof_lens, b2m_rng* rng, int* verdicts);
/* Phase split of the last b2m_verify_batch or b2m_verify_multi on this key (host wall-clock milliseconds around synchronised
 * work): {"decode_ms", "transcript_ms", "g2_set_ms", "msm_tables_ms", "msm_ms", "pairing_ms", "first_check_ms",
 * "bisection_ms", "checks", "keys", "g2_groups", "products", ...}.  g2_set_ms: assembling the call's G2 set from the keys'
 * prepared lines; keys: distinct keys of the call; products: pairing products over all checks. */
int b2m_verify_timings(const b2m_vk* vk, char* json, size_t cap);

#ifdef __cplusplus
}
#endif
#endif /* B2M_H */
