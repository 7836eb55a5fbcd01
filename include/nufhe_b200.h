/*
 * nufhe_b200.h -- C ABI of libnufhe_b200.so, the H100 (sm_90a) engine for the gate-bootstrapping hot
 * path of nucypher/nufhe, for programmable bootstrapping (lookup tables on small encrypted integers,
 * nb_bootstrap_lut_extract), for compressed cloud keys and ciphertexts, whose uniform masks are regenerated on the
 * device from a seed (nb_seeded_uniform_i32), for public-key encryption (nb_pk_prepare, nb_pk_encrypt), and for
 * packing results into GLWE samples (nb_pack_digits, nb_ntt_mac, nb_pack_finish), and for compact public-key
 * encryption (nb_compact_finish, nb_compact_extract).
 *
 * The reference has no FFI: its boundary is the set of Python call signatures listed in SURVEY.md
 * section 8(b).  Each entry point below replaces the device work behind one of them; the reference
 * file:line is cited next to it.  All array arguments are caller-owned, dense, C-contiguous DEVICE
 * pointers (torch `data_ptr()` / cudaMalloc) unless a name ends in `_host`; the library allocates only
 * inside nb_ctx (constant tables and per-call scratch).  Every call enqueues work on the context's
 * stream and returns without synchronising.  Return value: 0 on success, negative NB_E* otherwise;
 * nb_last_error() gives the message.  No torch types, no C++ types.
 *
 * Layouts (SURVEY.md Appendix C): LWE sample a:(B,n) int32, b:(B,) int32; TLWE accumulator (B,2,1024)
 * int32; reference bootstrap key (n,2,2,2,1024) uint64 = NTT(bk)*2^64 mod p in natural order; key-switch
 * key a:(1024,t,base,n) int32, b:(1024,t,base) int32, cv:(1024,t,base) float32.
 */
#ifndef NUFHE_B200_H
#define NUFHE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NB_OK 0
#define NB_EINVAL (-1)       /* bad argument (Python shim raises ValueError) */
#define NB_EUNSUPPORTED (-2) /* parameter set outside the built path (ValueError, as blind_rotate.py:37-86) */
#define NB_ECUDA (-3)        /* CUDA runtime error (RuntimeError) */

typedef struct nb_ctx nb_ctx;

/* Replaces the Reikna Thread of a nufhe.Context (api_high_level.py:153-181): binds (device, stream).
 * `stream` is a cudaStream_t (0 = default stream). */
int nb_ctx_create(int device, void *stream, nb_ctx **out);
void nb_ctx_destroy(nb_ctx *ctx);
const char *nb_last_error(const nb_ctx *ctx);
int nb_ctx_set_stream(nb_ctx *ctx, void *stream);
/* Pre-allocate the context's scratch (work queue and parked accumulators of the fused bootstrap, variance block sums
 * of the key switch) for launches of up to `batch` ciphertexts.  Calls within that size then allocate nothing, which
 * is what CUDA-graph capture of a gate circuit needs (reference counterpart: Reikna plans allocate their temporaries
 * when a computation is compiled, blind_rotate.py:245-246). */
int nb_ctx_reserve(nb_ctx *ctx, size_t batch);
int nb_ctx_synchronize(nb_ctx *ctx);          /* thread.synchronize() */
/* Library / device facts: sm count, kernel register counts etc. as a short text (for bench/profiles). */
const char *nb_build_info(void);

/* ---- transform: nufhe/transform/computation.py:28-99 `Transform` (natural order in and out) ---- */
/* ForwardTransform (polynomial_transform_ntt.py:120-124): int32 coefficients -> field, i32_conversion=True */
int nb_ntt_forward_i32(nb_ctx *ctx, const int32_t *in, uint64_t *out, size_t batch);
/* Transform(inverse=False, i32_conversion=False) */
int nb_ntt_forward_u64(nb_ctx *ctx, const uint64_t *in, uint64_t *out, size_t batch);
/* InverseTransform (polynomial_transform_ntt.py:127-131) */
int nb_ntt_inverse_i32(nb_ctx *ctx, const uint64_t *in, int32_t *out, size_t batch);
int nb_ntt_inverse_u64(nb_ctx *ctx, const uint64_t *in, uint64_t *out, size_t batch);

/* ---- field arithmetic: nufhe/transform/arithmetic.py:56-270 (element-wise; op codes below).
 * b may have b_period elements (broadcast, i % b_period) or be NULL for unary ops. */
#define NB_FF_ADD 0
#define NB_FF_SUB 1
#define NB_FF_MUL 2
#define NB_FF_MUL_PREPARED 3 /* a*b*2^-64, arithmetic.mako:355-419 */
#define NB_FF_PREPARE 4      /* a*2^64,    arithmetic.mako:336-352 */
#define NB_FF_LSH 5          /* a*2^b, b < 192, arithmetic.mako:465-1045 */
#define NB_FF_LSH_CONST 6    /* same result through the compile-time-shift code paths the transforms use */
int nb_ff_elementwise(nb_ctx *ctx, int op, const uint64_t *a, const uint64_t *b, uint64_t *out, size_t n,
                      size_t b_period);

/* ---- bootstrap key: BootstrapKey / TransformedTGswSampleArray (bootstrap.py:44-92, tgsw.py:99-130).
 * Re-lays `rows` reference rows (each 2*2*2*1024 uint64) into the engine's internal row format:
 * nb_bk_row_u64() uint64 per row (the 8 planes re-ordered and un-Montgomery-ed + 2 correction planes, then the
 * FP64 spectra of the 16-bit key halves).  Synchronises the context's stream: it records whether the key's
 * coefficients are centred 32-bit integers, which decides whether the throughput shape runs the FP64 step on it.
 * That choice is made per call and covers only the `rows` rows of that call: a launch takes the FP64 step only when
 * every key row it reads was prepared by one such call (a key assembled from several calls keeps the NTT step). */
size_t nb_bk_row_u64(void);
int nb_bk_prepare(nb_ctx *ctx, const uint64_t *bk_ref, uint64_t *bk_int, size_t rows);

/* ---- multi-bit bootstrap key (DESIGN.md section 14): key bits taken two at a time, group g = (s_2g, s_2g+1) has
 * 3 reference rows, row 3 g + p - 1 encrypting [s_2g = b0 and s_2g+1 = b1] for p = b0 + 2 b1 = 1, 2, 3.
 * Re-lays 3 * `groups` reference rows into nb_bk_multibit_row_u64() uint64 per row: the FP64 spectra of the 16-bit key
 * halves only.  Synchronises the context's stream.  NB_EINVAL if a coefficient is not a centred 32-bit integer.
 * The prepared range is registered on the context: nb_bootstrap_extract, nb_bootstrap_extract2,
 * nb_bootstrap_lut_extract and nb_bootstrap_glwe_lut_extract given a pointer into it run the multi-bit blind rotation
 * (n / 2 groups; n must be even), in the 2-ciphertext FP64 shape at every batch size; nb_blind_rotate and
 * nb_external_product return NB_EUNSUPPORTED for it. */
size_t nb_bk_multibit_row_u64(void);
int nb_bk_prepare_multibit(nb_ctx *ctx, const uint64_t *bk_ref, uint64_t *bk_mb, size_t groups);

/* ---- tgsw_transformed_external_mul (tgsw.py:165-172): accum (B,2,1024) <- bk[row] (x) accum ---- */
int nb_external_product(nb_ctx *ctx, int32_t *accum, const uint64_t *bk_int, size_t bk_row, size_t batch);

/* ---- BlindRotate_gpu (blind_rotate.py:262-281) without the key switch: explicit accumulator and bara.
 * out_a (B,1024), out_b (B,) receive the extracted samples; accum_out (optional) the rotated accumulators. */
int nb_blind_rotate(nb_ctx *ctx, const int32_t *accum, const int32_t *bara, const uint64_t *bk_int, size_t n,
                    int32_t *out_a, int32_t *out_b, int32_t *accum_out, size_t batch);

/* ---- bootstrap (bootstrap.py:206-229) fused with the gates' linear prologue (gates.py:108-115 etc.):
 * x = (0, c) + s1 * in1 + s2 * in2  (in2 may be NULL), then mod-switch, test vector, blind rotation and
 * sample extraction in one kernel.  Output: extracted LWE sample a:(B,1024), b:(B,). */
int nb_bootstrap_extract(nb_ctx *ctx, const int32_t *in1_a, const int32_t *in1_b, const int32_t *in2_a,
                         const int32_t *in2_b, int32_t c, int32_t s1, int32_t s2, int32_t mu,
                         const uint64_t *bk_int, size_t n, int32_t *out_a, int32_t *out_b, size_t batch);

/* ---- programmable bootstrap: the same prologue, x = (0, c) + s1 * in1 + s2 * in2, with an arbitrary test vector.
 * tv: 1024 int32 per vector, one for the batch (tv_stride 0) or one per ciphertext (tv_stride 1024); never NULL.
 * barb and every bara_i are rounded to multiples of 2^L (L = log2_outputs, 0..2), the accumulator starts as
 * (0, X^(2N - barb) * tv), and after the blind rotation the samples at indices j = 0 .. 2^L - 1 (coefficient j of the
 * phase: extraction after a rotation by X^(-j)) go to rows c * 2^L + j.  Output: out_a (B * 2^L, 1024),
 * out_b (B * 2^L,).  NB_EINVAL for a NULL tv, a stride other than 0 / 1024 or L outside 0..2.  The key switch of
 * the B * 2^L samples that usually follows needs nb_ctx_reserve(B * 2^L) before a graph capture. */
int nb_bootstrap_lut_extract(nb_ctx *ctx, const int32_t *in1_a, const int32_t *in1_b, const int32_t *in2_a,
                             const int32_t *in2_b, int32_t c, int32_t s1, int32_t s2, const int32_t *tv,
                             size_t tv_stride, int log2_outputs, const uint64_t *bk_int, size_t n, int32_t *out_a,
                             int32_t *out_b, size_t batch);

/* Two bootstraps in one launch (gate_mux, gates.py:638-655): job A on ciphertexts [0, B), job B on [B, 2B);
 * out_a (2B,1024), out_b (2B,).  Halves the latency of small-batch MUX gates. */
int nb_bootstrap_extract2(nb_ctx *ctx, const int32_t *a1_a, const int32_t *a1_b, const int32_t *a2_a,
                          const int32_t *a2_b, int32_t a_c, int32_t a_s1, int32_t a_s2, const int32_t *b1_a,
                          const int32_t *b1_b, const int32_t *b2_a, const int32_t *b2_b, int32_t b_c, int32_t b_s1,
                          int32_t b_s2, int32_t mu, const uint64_t *bk_int, size_t n, int32_t *out_a, int32_t *out_b,
                          size_t batch);

/* ---- lwe_keyswitch (lwe.py:311-322): res = keyswitch((0, c) + src1 + src2), src2 may be NULL.
 * res_cv may be NULL. */
int nb_keyswitch(nb_ctx *ctx, const int32_t *src1_a, const int32_t *src1_b, const int32_t *src2_a,
                 const int32_t *src2_b, int32_t c, const int32_t *ks_a, const int32_t *ks_b, const float *ks_cv,
                 size_t in_size, size_t n, int t, int log2_base, int32_t *res_a, int32_t *res_b, float *res_cv,
                 size_t batch);

/* ---- the key switch as a tensor-core GEMM (DESIGN.md section 4).  nb_ks_prepare lays a key-switch key with in = 1024,
 * n = 500, t = 8 and base 4 into the byte planes that keyswitch_mma_kernel streams (`out`: nb_ks_prepared_bytes()
 * bytes, 16-byte aligned, about 50 MB), and registers them on the context under (ks_a, ks_b).  From then on
 * nb_keyswitch with that ks_a and ks_b runs batches from a measured threshold up (environment variable
 * NUFHE_B200_KS_MMA_MIN, read at context creation) as one exact u8 x u8 -> s32 wgmma GEMM; results and variances are
 * bit-identical to the other path.  Rows d = 0 are left out of the GEMM: a key whose d = 0 rows are not all zero is
 * prepared but not registered, and keeps the other path.  *registered (may be NULL) is 1 when the key was
 * registered.  Prepare again after changing the key, and call nb_ks_forget(ctx, ks_a) before freeing `out` or the
 * key.  NB_EUNSUPPORTED for other parameters, NB_EINVAL for a NULL pointer or a misaligned `out`. */
size_t nb_ks_prepared_bytes(void);
int nb_ks_prepare(nb_ctx *ctx, const int32_t *ks_a, const int32_t *ks_b, uint8_t *out, size_t in_size, size_t n, int t,
                  int log2_base, int *registered);
int nb_ks_forget(nb_ctx *ctx, const int32_t *ks_a);

/* ---- multi-key calls (DESIGN.md section 17): one launch over ciphertexts of several cloud keys ("tenants").
 * Each takes the arguments of the single-key call of the same name, with the key replaced by HOST arrays of one entry
 * per tenant (`tenants` entries): the key pointers, and counts[t], the number of consecutive ciphertexts of the batch
 * that belong to tenant t, in tenant order; the counts add up to `batch` (for extract2 they apply to each job, so job
 * A is [0, batch) and job B [batch, 2 batch), both split by the same counts; for the key switch of the 2^L samples of
 * nb_mk_bootstrap_lut_extract pass counts * 2^L).  A count may be 0.  Every output row is bit-identical to the
 * single-key call on that tenant's segment with that tenant's key.  The bootstrap runs in the 2-ciphertext FP64 shape
 * at every batch size; every key must lie inside one engine key prepared by nb_bk_prepare on this context with FP64
 * spectra.  The key switch runs each tenant whose segment would take the tensor-core GEMM in nb_keyswitch exactly as
 * there, and all the others in one launch of the gather kernel whose tiles never cross a tenant boundary; it takes
 * in = 1024, n = 500, t = 8, base 4 only.  The library uploads the per-ciphertext tenant table and the tile table into
 * context scratch; these calls are not for graph capture.
 * NB_EINVAL for a NULL argument, counts that do not add up to `batch`, or a key that is not inside a prepared engine
 * key of this context; NB_EUNSUPPORTED for a multi-bit key, a context with the FP64 step disabled (NUFHE_B200_FFT=0),
 * an LWE dimension out of range or other key-switch sizes. */
int nb_mk_bootstrap_extract(nb_ctx *ctx, const int32_t *in1_a, const int32_t *in1_b, const int32_t *in2_a,
                            const int32_t *in2_b, int32_t c, int32_t s1, int32_t s2, int32_t mu,
                            const uint64_t *const *bk_int_host, const size_t *counts_host, size_t tenants, size_t n,
                            int32_t *out_a, int32_t *out_b, size_t batch);
int nb_mk_bootstrap_extract2(nb_ctx *ctx, const int32_t *a1_a, const int32_t *a1_b, const int32_t *a2_a,
                             const int32_t *a2_b, int32_t a_c, int32_t a_s1, int32_t a_s2, const int32_t *b1_a,
                             const int32_t *b1_b, const int32_t *b2_a, const int32_t *b2_b, int32_t b_c, int32_t b_s1,
                             int32_t b_s2, int32_t mu, const uint64_t *const *bk_int_host, const size_t *counts_host,
                             size_t tenants, size_t n, int32_t *out_a, int32_t *out_b, size_t batch);
int nb_mk_bootstrap_lut_extract(nb_ctx *ctx, const int32_t *in1_a, const int32_t *in1_b, const int32_t *in2_a,
                                const int32_t *in2_b, int32_t c, int32_t s1, int32_t s2, const int32_t *tv,
                                size_t tv_stride, int log2_outputs, const uint64_t *const *bk_int_host,
                                const size_t *counts_host, size_t tenants, size_t n, int32_t *out_a, int32_t *out_b,
                                size_t batch);
int nb_mk_keyswitch(nb_ctx *ctx, const int32_t *src1_a, const int32_t *src1_b, const int32_t *src2_a,
                    const int32_t *src2_b, int32_t c, const int32_t *const *ks_a_host, const int32_t *const *ks_b_host,
                    const float *const *ks_cv_host, const size_t *counts_host, size_t tenants, size_t in_size, size_t n,
                    int t, int log2_base, int32_t *res_a, int32_t *res_b, float *res_cv, size_t batch);
/* The multi-key forms of tree LUTs and result packing (DESIGN.md section 18), with the conventions above.
 * nb_mk_bootstrap_glwe_lut_extract: nb_bootstrap_glwe_lut_extract with per-tenant keys and counts, as
 *     nb_mk_bootstrap_extract (same refusals).
 * nb_mk_tree_keyswitch: nb_tree_keyswitch with per-tenant planes (nb_tree_prepare) and counts of rows; a CTA covers up
 *     to 256 rows of one tenant.  NB_EINVAL also for a NULL planes pointer and the sizes nb_tree_keyswitch refuses.
 * nb_mk_ntt_mac: nb_ntt_mac with per-tenant key spectra and group_counts[t], the number of consecutive groups of x
 *     that belong to tenant t (they add up to `groups`).  NB_EINVAL also for a NULL key and the sizes nb_ntt_mac
 *     refuses. */
int nb_mk_bootstrap_glwe_lut_extract(nb_ctx *ctx, const int32_t *in_a, const int32_t *in_b, const int32_t *tv,
                                     const uint64_t *const *bk_int_host, const size_t *counts_host, size_t tenants,
                                     size_t n, int32_t *out_a, int32_t *out_b, size_t batch);
int nb_mk_tree_keyswitch(nb_ctx *ctx, const int32_t *a, const uint8_t *const *planes_host, const size_t *counts_host,
                         size_t tenants, size_t n, int mask_size, int32_t *out, size_t rows);
int nb_mk_ntt_mac(nb_ctx *ctx, const uint64_t *x, const uint64_t *const *key_host, const size_t *group_counts_host,
                  size_t tenants, uint64_t *out, size_t rows, size_t outs, size_t groups);
/* Expansion of compressed cloud keys into slots of the multi-key machine (DESIGN.md section 19).  seeds_host holds 8
 * words per tenant, the seed of its compressed key; the other per-tenant arrays are HOST arrays of device pointers.
 * Neither call allocates (beyond the multi-key scratch) or synchronises.
 * nb_mk_bk_expand: slot t (n rows of nb_bk_row_u64() uint64) receives the FP64 part of the engine key of the bootstrap
 *     key whose masks are the stream (seed t, nonce 1) laid out (n, k+1, l, k, N) (nb_seeded_uniform_i32) and whose
 *     bodies are bodies_host[t] (n, k+1, l, N) int32: word for word what nb_bk_prepare stores there for that key.  The
 *     NTT planes of the rows are not written, so the slot is registered for the nb_mk_* bootstraps only (it replaces any
 *     earlier registration of the range); nb_mk_slot_release(ctx, slot) drops it, before the slot's memory is freed.
 *     k = 1, l = 2, N = 1024 and 1 <= n <= 1024 only (NB_EUNSUPPORTED otherwise).
 * nb_mk_ks_expand: ks_a_host[t] (in, t, base, n) int32 receives the masks of the stream (seed t, nonce 2) laid out
 *     (in, t, base-1, n) in its rows h >= 1 and zeros in its rows h = 0, as CompressedCloudKey.decompress() lays them
 *     out; a GEMM registration (nb_ks_prepare) of that ks_a is dropped.  in = 1024, n = 500, t = 8, base 4 only
 *     (NB_EUNSUPPORTED otherwise).
 * NB_EINVAL for a NULL pointer; tenants = 0 is a no-op. */
int nb_mk_bk_expand(nb_ctx *ctx, const uint32_t *seeds_host, const int32_t *const *bodies_host,
                    uint64_t *const *slots_host, size_t tenants, size_t n, int mask_size, int decomp_length,
                    size_t poly_degree);
int nb_mk_ks_expand(nb_ctx *ctx, const uint32_t *seeds_host, int32_t *const *ks_a_host, size_t tenants, size_t in_size,
                    int t, int log2_base, size_t n);
int nb_mk_slot_release(nb_ctx *ctx, const uint64_t *slot);

/* ---- LweLinear / LweNoiselessTrivial (lwe.py:346-422): res = (0, c) + s1 * x1 + s2 * x2 ------- */
int nb_lwe_affine(nb_ctx *ctx, int32_t *res_a, int32_t *res_b, const int32_t *x1_a, const int32_t *x1_b,
                  const int32_t *x2_a, const int32_t *x2_b, int32_t c, int32_t s1, int32_t s2, size_t batch,
                  size_t n);

/* ---- the separate steps of the multi-kernel bootstrap (bootstrap.py:96-196), `single_kernel_bootstrap=False` ---- */
/* ShiftTorusPolynomial (polynomials.py:90-104, polynomials_gpu.mako:18-77).  mode NB_SHIFT_INVERT: result =
 * X^(2N - power) * source (shift_tp_inverted_power); NB_SHIFT_MINUS_ONE: (X^power - 1) * source
 * (shift_tp_minus_one_power_from_array / tlwe_shift_polynomials); NB_SHIFT_PLAIN: X^power * source.
 * source/result: (polys, N) int32, N = 2^n_log2.  Polynomial p uses
 * powers[(p / polys_per_power) * powers_stride + power_idx]. */
#define NB_SHIFT_INVERT 0
#define NB_SHIFT_MINUS_ONE 1
#define NB_SHIFT_PLAIN 2
int nb_shift_torus_polynomial(nb_ctx *ctx, int32_t *result, const int32_t *source, const int32_t *powers,
                              size_t powers_stride, size_t power_idx, int polys_per_power, int mode, int n_log2,
                              size_t polys);
/* tlwe_noiseless_trivial (tlwe.py:156-158): acc (B, k+1, N) = (0, .., 0, mu (B, N)); cv (B,) = 0, one variance per
 * sample (may be NULL) */
int nb_tlwe_noiseless_trivial(nb_ctx *ctx, int32_t *acc, float *cv, const int32_t *mu, int mask_size, int n_log2,
                              size_t batch);
/* tlwe_extract_lwe_samples (tlwe.py:161-165): out_a (B, k*N), out_b (B,) from acc (B, k+1, N) */
int nb_tlwe_extract_lwe_samples(nb_ctx *ctx, int32_t *out_a, int32_t *out_b, const int32_t *acc, int mask_size,
                                int n_log2, size_t batch);
/* t32_to_phase (numeric_functions.py:34-36, kernel numeric_functions_gpu.py:39-77): the mod-switch of bootstrap()
 * (bootstrap.py:216-219) as a separate step; mspace_size must divide 2^32 */
int nb_t32_to_phase(nb_ctx *ctx, int32_t *out, const int32_t *in, size_t n, uint32_t mspace_size);
/* The external product of the multi-kernel path step by step (TGswTransformedExternalMul, tgsw_gpu.py:110-169), for
 * any TLWE mask size k and decomposition length l -- the fused kernel covers k = 1, l = 2 only:
 * decompose -> nb_ntt_forward_i32 -> MAC -> nb_ntt_inverse_i32.
 * nb_tgsw_decompose (tgsw_gpu.py:31-54): out (polys, l, N) from in (polys, N); offset = TGswParams.offset.
 * nb_tgsw_mac (tgsw_gpu.py:58-107): out (B, k+1, 1024) = sum_{mi,j} mul_prepared(tr (B, k+1, l, 1024),
 * bk_row (k+1, l, k+1, 1024)), bk_row in the reference's layout (natural order, Montgomery form). */
int nb_tgsw_decompose(nb_ctx *ctx, int32_t *out, const int32_t *in, size_t polys, int decomp_length, int bs_log2_base,
                      int32_t offset, int n_log2);
int nb_tgsw_mac(nb_ctx *ctx, uint64_t *out, const uint64_t *tr, const uint64_t *bk_row, size_t batch, int mask_size,
                int decomp_length);
/* tlwe_add_to (tlwe.py:173-175): res += src (int32 wrap-around, n elements); variances (n_cv floats, may be NULL) */
int nb_tlwe_add_to(nb_ctx *ctx, int32_t *res, const int32_t *src, size_t n, float *res_cv, const float *src_cv,
                   size_t n_cv);

/* LweEncrypt / LweDecrypt (lwe_gpu.py:186-284, kernels lwe_gpu.mako:205-262; lwe.py:325-343): the wrap-around dot
 * product of LWE masks a (B, n) with the binary key (n),
 *     out[i] = add1[i] (+ add2[i]) + sign * <a[i, :], key>       (add1, add2 may be NULL)
 * encrypt: out = b, add1 = messages, add2 = noises_b, sign = +1;  decrypt phase: add1 = b, sign = -1. */
int nb_lwe_dot(nb_ctx *ctx, int32_t *out, const int32_t *a, const int32_t *key, const int32_t *add1,
               const int32_t *add2, int32_t sign, size_t batch, size_t n);
/* MakeLweKeyswitchKey (lwe_gpu.py:63-124, kernel lwe_gpu.mako:18-56; lwe.py:265-295): ks_a (in, t, base, n),
 * ks_b / ks_cv (in, t, base) from in_key (in), out_key (n), noises_a (in, t, base-1, n), noises_b (in, t, base-1):
 * row h = 0 is zero, row h encrypts in_key[i] * h * 2^(32 - (j+1) log2_base) with variance noise_variance. */
int nb_make_keyswitch_key(nb_ctx *ctx, int32_t *ks_a, int32_t *ks_b, float *ks_cv, const int32_t *in_key,
                          const int32_t *out_key, const int32_t *noises_a, const int32_t *noises_b, size_t in_size,
                          size_t n, int t, int log2_base, float noise_variance);

/* ---- seeded masks of compressed keys and ciphertexts (DESIGN.md section 10; no reference counterpart):
 * out[i] = word (first + i) of the ChaCha20 keystream (seed_host: 8 words, nonce), i < count, as int32.
 * The stream is the RFC 8439 block function in the original 64-bit-counter layout (state words 12-13 the block
 * counter, 14-15 the nonce); word w is word w % 16 of block w / 16, so `first` may start mid-block.  seed_host is a
 * HOST pointer.  NB_EINVAL for a NULL seed or output and for first + count past 2^64. */
int nb_seeded_uniform_i32(nb_ctx *ctx, const uint32_t *seed_host, uint64_t nonce, uint64_t first, int32_t *out,
                          size_t count);

/* ---- public-key encryption (DESIGN.md section 11; no reference counterpart).  A public key is m LWE encryptions of 0,
 * a (m, n) int32 and b (m,) int32; encrypting B messages is (a, b) = R [A | b_pk] + (0, mu) with R binary (B, m).
 * nb_pk_prepare lays W = [A | b | 1] (m x (n+2), columns padded to a multiple of 8) into 4 byte planes, plane p
 * column-major: byte p of W[k][col] at ((p * npad + col) * m + k); `planes` holds nb_pk_planes_bytes(m, n) bytes
 * (0 for an n the library rejects).
 * nb_pk_encrypt: r_bits (B, m/32) uint32, bit i of row c = bit i % 32 of word (c, i / 32);
 *     out_a[c] = sum_i r_ci A_i,  out_b[c] = mus[c] + sum_i r_ci b_i  (mod 2^32),
 *     out_cv[c] = float(popcount(r_c)) * row_variance,
 * one exact u8 x u8 -> s32 tensor-core GEMM (mma.sync m16n8k32).  NB_EINVAL for a NULL pointer, for m not a positive
 * multiple of 32 or with m * 255 >= 2^31 (the sums would not be exact), and for n = 0; batch = 0 is a no-op. */
size_t nb_pk_planes_bytes(size_t m, size_t n);
int nb_pk_prepare(nb_ctx *ctx, const int32_t *a, const int32_t *b, size_t m, size_t n, uint8_t *planes);
int nb_pk_encrypt(nb_ctx *ctx, const uint32_t *r_bits, const uint8_t *planes, size_t m, size_t n, const int32_t *mus,
                  float row_variance, int32_t *out_a, int32_t *out_b, float *out_cv, size_t batch);

/* ---- result packing (DESIGN.md section 12; no reference counterpart).  B LWE samples under the n-word key become
 * G = ceil(B / 1024) GLWE samples (k + 1 polynomials of N = 1024 coefficients): input c goes to group c / 1024, slot
 * c % 1024.  The steps: nb_pack_digits, nb_ntt_forward_i32 of the digits, nb_ntt_mac with the spectra of the packing
 * key, nb_ntt_inverse_i32, nb_pack_finish.
 * nb_pack_digits: a (B, n) int32 -> digits (G, 2 n, N) int32; row 2 i + j of group g holds at coefficient p the digit j
 *     of a[g N + p][i]: with w = a + 2^15 + 2^23 + 2^31 (mod 2^32), d_0 = (w >> 24) - 128, d_1 = ((w >> 16) & 255) - 128.
 *     Empty slots of the last group are 0.  NB_EINVAL for a NULL pointer, n = 0 or n > 2^20, and G > 2047.
 * nb_ntt_mac: out (G, U, N) = sum_{r < R} x (G, R, N) . key (R, U, N), element-wise products of plain-form (not
 *     Montgomery) field elements, out canonical.  NB_EINVAL for a NULL pointer, R = 0, U = 0, R > 2^24 or U > 2^16.
 * nb_pack_finish: c (G, k + 1, N) int32, the inverse transform of the MAC, and the bodies b (B,) int32 ->
 *     out (G, k + 1, N) uint16: round_16(-c) for polynomials u < k, round_16(b[g N + p] - c) at coefficient p of the
 *     body (b = 0 in empty slots), round_16(x) = (x + 2^15) >> 16 on the 32-bit x.  NB_EINVAL for a NULL pointer and
 *     k < 1.
 * batch / groups = 0 is a no-op for all three. */
int nb_pack_digits(nb_ctx *ctx, const int32_t *a, size_t n, int32_t *digits, size_t batch);
int nb_ntt_mac(nb_ctx *ctx, const uint64_t *x, const uint64_t *key, uint64_t *out, size_t rows, size_t outs,
               size_t groups);
int nb_pack_finish(nb_ctx *ctx, const int32_t *c, const int32_t *b, int mask_size, uint16_t *out, size_t batch);

/* ---- tree-based programmable bootstrapping (DESIGN.md section 13; no reference counterpart).  A lookup table on D
 * digits is evaluated one digit at a time: the LWE outputs of one level become GLWE test vectors under the bootstrap
 * key's GLWE key S (k polynomials of N = 1024), which the next level blind-rotates by the next digit.
 * The tree key T: n t = 2 n rows, row i t + j a GLWE encryption under S of the constant s_i g_j (g = 2^24, 2^16), as
 * masks (n, t, k, N) and bodies (n, t, N) int32.
 * nb_tree_prepare lays T ((n t) x (k+1) N, rows padded with zeros to kpad = n t rounded up to 32) into 4 byte planes,
 *     plane p column-major: byte p of T[row][col] at ((p * (k+1) N + col) * kpad + row); `planes` holds
 *     nb_tree_planes_bytes(n, k) bytes (0 for sizes the library rejects).
 * nb_tree_keyswitch: a (R, n) int32 LWE masks -> out (R, k+1, N) int32, V = sum_ij d_ij(a_r) T_ij mod 2^32 with the
 *     signed digits d_ij of nb_pack_digits (round_16(a_i) = d_i0 g_0 + d_i1 g_1), one exact s8 x u8 -> s32
 *     tensor-core GEMM (mma.sync m16n8k32) per byte plane.
 * nb_tree_assemble: v (count, 2^bits, k+1, N) and the LWE bodies b (count, 2^bits) -> tv (count, k+1, N),
 *     tv_u = sum_m X^(o_m) (1 + X + ... + X^(box - 1)) G_m,u (negacyclic, mod 2^32), box = N >> bits,
 *     o_m = m box - box / 2, G_m,u = -v_m,u for u < k and b_m X^0 - v_m,k for u = k.
 * NB_EINVAL for a NULL pointer, n = 0 or kpad * 128 * 255 >= 2^31 (the sums would not be exact), a mask size outside
 * 1..16 and bits outside 1..2; rows / count = 0 is a no-op. */
size_t nb_tree_planes_bytes(size_t n, int mask_size);
int nb_tree_prepare(nb_ctx *ctx, const int32_t *masks, const int32_t *body, size_t n, int mask_size, uint8_t *planes);
int nb_tree_keyswitch(nb_ctx *ctx, const int32_t *a, const uint8_t *planes, size_t n, int mask_size, int32_t *out,
                      size_t rows);
int nb_tree_assemble(nb_ctx *ctx, const int32_t *v, const int32_t *b, int bits, int mask_size, int32_t *tv,
                     size_t count);
/* The programmable bootstrap of one LWE input (in_a (B, n), in_b (B,)) with a per-ciphertext GLWE test vector
 * tv (B, 2, 1024) (k = 1, the fused kernel's parameter set): the accumulator starts as X^(2N - barb) * (tv_0, tv_1)
 * instead of (0, X^(2N - barb) * tv), L = 0.  Output: out_a (B, 1024), out_b (B,).  NB_EINVAL for a NULL pointer;
 * batch = 0 is a no-op. */
int nb_bootstrap_glwe_lut_extract(nb_ctx *ctx, const int32_t *in_a, const int32_t *in_b, const int32_t *tv,
                                  const uint64_t *bk_int, size_t n, int32_t *out_a, int32_t *out_b, size_t batch);

/* ---- encrypted-index table lookups (DESIGN.md section 15; no reference counterpart).  A query holds m TGSW selectors
 * (the client-encrypted bits of an index, N = 1024, k = 1, l = 2, Bg = 2^10), each (2, 2, 2, N) int32 in the layout of
 * a bootstrap-key row.  All three run the FP64 CMux step; GLWE samples are (2, N) int32.
 * nb_index_prepare: `rows` selector rows -> spectra (rows, BK_FFT_U64) uint64 (nb_bk_multibit_row_u64() words per row,
 *     the layout nb_bk_prepare_multibit stores).
 * nb_index_cmux_level: out[q][i] = in[q][2i] + sel[q] (x) (in[q][2i+1] - in[q][2i]) for i < nodes, q < queries; in[q]
 *     starts in_query_stride int32 words after in[q-1] (0: one plaintext level shared by every query), sel[q]
 *     sel_query_stride uint64 words after sel[q-1]; out (queries, nodes, 2, N).
 * nb_index_rotate_extract: for j < min(bits, 10), ACC <- ACC + sel_j[q] (x) ((X^(-2^j) - 1) ACC), sel_j[q] = sel +
 *     q sel_query_stride + j BK_FFT_U64, then sample extraction.  bits >= 10: `columns` accumulators per query
 *     (consecutive, acc_query_stride words between queries), each extracted at coefficient 0.  bits < 10: one
 *     accumulator per query, extracted at coefficients w 2^bits, w < columns.  Column w of query q goes to row
 *     w * queries + q of out_a (columns * queries, N) and out_b (columns * queries).
 * NB_EINVAL for a NULL pointer, bits outside 1..20, columns = 0, columns 2^bits > N for bits < 10, or a batch beyond
 * the grid; rows / nodes / queries = 0 is a no-op. */
int nb_index_prepare(nb_ctx *ctx, const int32_t *ggsw, size_t rows, uint64_t *spectra);
int nb_index_cmux_level(nb_ctx *ctx, const int32_t *in, size_t in_query_stride, const uint64_t *sel,
                        size_t sel_query_stride, int32_t *out, size_t nodes, size_t queries);
int nb_index_rotate_extract(nb_ctx *ctx, const int32_t *acc, size_t acc_query_stride, const uint64_t *sel,
                            size_t sel_query_stride, int bits, size_t columns, int32_t *out_a, int32_t *out_b,
                            size_t queries);

/* The same two levels with one table per query (encrypted tables, DESIGN.md section 20): `tables` holds table_count
 * tables, table_stride int32 words apart, and query q reads table table_ids_host[q] (a host array of `queries` entries,
 * uploaded by the call) where the calls above read in + q in_query_stride.  They serve the level that first reads a
 * table: nb_index_cmux_level_indirect for bits > 10 (each table 2 nodes GLWE samples), nb_index_rotate_extract_indirect
 * for bits <= 10 (each table `columns` accumulators for bits = 10, one below).  NB_EINVAL as above, and for an id
 * >= table_count or a stride shorter than a table. */
int nb_index_cmux_level_indirect(nb_ctx *ctx, const int32_t *tables, size_t table_stride, size_t table_count,
                                 const uint32_t *table_ids_host, const uint64_t *sel, size_t sel_query_stride,
                                 int32_t *out, size_t nodes, size_t queries);
int nb_index_rotate_extract_indirect(nb_ctx *ctx, const int32_t *tables, size_t table_stride, size_t table_count,
                                     const uint32_t *table_ids_host, const uint64_t *sel, size_t sel_query_stride,
                                     int bits, size_t columns, int32_t *out_a, int32_t *out_b, size_t queries);

/* ---- oblivious writes into encrypted tables (DESIGN.md section 21; no reference counterpart): the transpose of a
 * lookup, on the same FP64 CMux step and selector spectra.
 * nb_index_write_assemble: the delta of every query, (0, b) - V: v (queries, columns, 2, N) (the nb_tree_keyswitch
 *     output of the values' masks; NULL for trivial values, V = 0) and b (queries, columns) -> out (queries, A, 2, N),
 *     A = columns for bits >= 10 (one sample per column), A = 1 below (column w times X^(w 2^bits)).
 * nb_index_write_rotate: for j < min(bits, 10), ACC <- ACC + sel_j[q] (x) ((X^(+2^j) - 1) ACC) on each of the A deltas
 *     of query q (sel_j[q] as for nb_index_rotate_extract).  bits > 10: the samples go to out (queries, A, 2, N) and acc
 *     must be NULL.  bits <= 10: sample c of query q is added (mod 2^32) into sample c of table table_ids_host[q] of
 *     acc (acc_count tables of int32 GLWE samples, acc_stride words apart; table_ids_host NULL: one table), out unused.
 * nb_index_demux_level: node y of in (queries, nodes, 2, N) becomes (y - sel[q] (x) y, sel[q] (x) y) at nodes 2i, 2i+1
 *     of out (queries, 2 nodes, 2, N), or, with acc, is added into samples 2i, 2i+1 of the query's table (the last
 *     level, bit 10).
 * Adds are atomic, and sums mod 2^32 do not depend on their order.  NB_EINVAL for a NULL pointer, bits outside 1..20,
 * columns 2^bits > N below 10 bits, acc given or missing against the rule above, a stride shorter than a table, an id
 * >= acc_count or several tables without ids; queries = 0 is a no-op. */
int nb_index_write_assemble(nb_ctx *ctx, const int32_t *v, const int32_t *b, int bits, size_t columns, int32_t *out,
                            size_t queries);
int nb_index_write_rotate(nb_ctx *ctx, const int32_t *delta, const uint64_t *sel, size_t sel_query_stride, int bits,
                          size_t columns, int32_t *out, int32_t *acc, size_t acc_stride, size_t acc_count,
                          const uint32_t *table_ids_host, size_t queries);
int nb_index_demux_level(nb_ctx *ctx, const int32_t *in, const uint64_t *sel, size_t sel_query_stride, int32_t *out,
                         int32_t *acc, size_t acc_stride, size_t acc_count, const uint32_t *table_ids_host,
                         size_t nodes, size_t queries);

/* ---- compact public-key encryption (DESIGN.md section 16; no reference counterpart).  B messages go into
 * G = ceil(B / 1024) GLWE samples under the bootstrap key's GLWE key S (k + 1 polynomials of N = 1024 coefficients),
 * message c in group c / 1024, slot c % 1024, every coefficient rounded to 16 bits.  Encryption: nb_ntt_forward_i32 of
 * the binary polynomials r (G, N), nb_ntt_mac with the spectra of the compact public key (1, k + 1, N),
 * nb_ntt_inverse_i32, nb_compact_finish.  Expansion: nb_compact_extract, then nb_keyswitch with the cloud key.
 * nb_compact_finish: c (G, k + 1, N) int32 (the products), e1 (G, k, N), e2 (G, N) and the messages mus (B,) int32 ->
 *     out (G, k + 1, N) uint16: round_16(c_u + e1_u) for polynomials u < k, round_16(c_k + e2 + mus[g N + p]) at an
 *     occupied coefficient p of the body and 0 at an empty one, round_16(x) = (x + 2^15) >> 16 on the 32-bit x.
 *     NB_EINVAL for a NULL pointer and k < 1.
 * nb_compact_extract: data (ceil(rows / 1024), k + 1, N) uint16 -> out_a (rows, k N), out_b (rows,) int32: with
 *     x' = x << 16, row c = g N + p holds a[u N + j] = A'_u[p - j] for j <= p and -A'_u[N + p - j] for j > p, and
 *     b = body'[p].  NB_EINVAL for a NULL pointer, k < 1, data not 8-byte or out_a not 16-byte aligned, and more than
 *     65535 groups.
 * batch / rows = 0 is a no-op for both. */
int nb_compact_finish(nb_ctx *ctx, const int32_t *c, const int32_t *e1, const int32_t *e2, const int32_t *mus,
                      int mask_size, uint16_t *out, size_t batch);
int nb_compact_extract(nb_ctx *ctx, const uint16_t *data, int mask_size, int32_t *out_a, int32_t *out_b, size_t rows);

#ifdef __cplusplus
}
#endif
#endif
