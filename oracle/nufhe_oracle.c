/*
 * nufhe_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * A plain-C CPU restatement of the hot path of nucypher/nufhe (TFHE gate bootstrapping on the
 * NTT transform).  It exists only so that tests/, __graft_entry__.smoke() and the cpu_baseline /
 * --impl reference legs of bench.py can check and time-compare the CUDA implementation; nothing under
 * nufhe_b200/ may import, link or execute it.
 *
 * Parity pin: every function here is checked against the reference's own NumPy closures
 * (nufhe/<module>_cpu.py, nufhe/transform/ntt_cpu.py) by tests/golden/make_golden.py, whose outputs are
 * committed under tests/golden/ and re-checked by tests/test_oracle.py.
 *
 * Each function cites the reference file:line it restates (paths relative to /root/reference).
 * Arithmetic is exact: Torus32 = wrapping int32, field = Z_p with p = 2^64 - 2^32 + 1.
 *
 * Default scheme parameters only (nufhe/api_low_level.py:49-56): N=1024, k=1, l=2, Bg=2^10.
 * LWE sizes and key-switch parameters are run-time arguments.
 */
#include <stdint.h>
#include <stddef.h>
#include <stdlib.h>
#include <string.h>

typedef uint64_t u64;
typedef uint32_t u32;
typedef int32_t i32;
typedef unsigned __int128 u128;

#define P 0xffffffff00000001ULL          /* nufhe/transform/ntt_cpu.py:23 */
#define NPOLY 1024                       /* nufhe/api_low_level.py:49 */
#define MASK_K 1                         /* api_low_level.py:44 (tlwe_mask_size) */
#define DECOMP_L 2                       /* api_low_level.py:52 */
#define BS_LOG2_BASE 10                  /* api_low_level.py:53 */
#define ROOT_GEN 0xa70dc47e4cbdf43fULL   /* ntt_cpu.py:109 */
#define R_INV 0xfffffffe00000001ULL      /* 2^-64 mod p, polynomial_transform_ntt.py:66 */

/* ------------------------------------------------------------------ Z_p ---------------------- */

/* GaloisNumber.__add__ / __sub__ / __mul__, ntt_cpu.py:29-36 (operands canonical) */
static inline u64 ff_add(u64 a, u64 b) { u128 s = (u128)a + b; return (u64)(s >= P ? s - P : s); }
static inline u64 ff_sub(u64 a, u64 b) { return a >= b ? a - b : (u64)((u128)a + P - b); }
/* (a*b) mod p.  The 128-bit product is folded with 2^64 = 2^32-1 and 2^96 = -1 (mod p), the same
 * identities the reference uses (arithmetic.mako:200-207); orc_selftest() checks it against `%`. */
static inline u64 ff_reduce128(u128 x)
{
    u64 lo = (u64)x, hi = (u64)(x >> 64);
    u64 hi_hi = hi >> 32, hi_lo = hi & 0xffffffffULL;
    u64 t0 = lo - hi_hi;
    if (lo < hi_hi) t0 -= 0xffffffffULL;            /* wrapped by 2^64 = 2^32-1 */
    u64 t1 = (hi_lo << 32) - hi_lo;                 /* hi_lo * (2^32-1) */
    u64 r = t0 + t1;
    if (r < t1) r += 0xffffffffULL;
    return r >= P ? r - P : r;
}
static inline u64 ff_mul(u64 a, u64 b) { return ff_reduce128((u128)a * b); }
static inline u64 ff_mul_slow(u64 a, u64 b) { return (u64)(((u128)a * b) % P); }

static u64 ff_pow(u64 a, u64 e)          /* ntt_cpu.py:41-54 */
{
    u64 r = 1;
    while (e) { if (e & 1) r = ff_mul(r, a); a = ff_mul(a, a); e >>= 1; }
    return r;
}
static u64 ff_inv(u64 a) { return ff_pow(a, P - 2); }   /* ntt_cpu.py:56-57 */

/* transformed_space_mul_prepared_ref, polynomial_transform_ntt.py:65-69: a*b*2^-64 mod p */
static inline u64 ff_mul_prepared(u64 a, u64 b) { return ff_mul(ff_mul(a % P, b % P), R_INV); }

/* prepare_for_mul_cpu, transform/arithmetic.py:172-195: x * 2^64 mod p */
static inline u64 ff_prepare_for_mul(u64 x) { return (u64)((((u128)(x % P)) << 64) % P); }

/* int32 -> field: ntt.mako:395-399 (x>=0 -> x, x<0 -> p-|x|), same as GaloisNumber(int) ntt_cpu.py:27 */
static inline u64 ff_from_i32(i32 x) { return x >= 0 ? (u64)x : P - (u64)(-(int64_t)x); }

/* field -> int32: ntt_cpu.py:74-80 (as patched for NumPy 2, SURVEY Appendix D), ntt.mako:402-408 */
static inline i32 ff_to_i32(u64 v) { return (i32)((u32)v - (u32)(v > P / 2)); }

void orc_ff_mul(u64 *out, const u64 *a, const u64 *b, size_t n)
{ for (size_t i = 0; i < n; i++) out[i] = ff_mul(a[i] % P, b[i] % P); }
void orc_ff_add(u64 *out, const u64 *a, const u64 *b, size_t n)
{ for (size_t i = 0; i < n; i++) out[i] = ff_add(a[i] % P, b[i] % P); }
void orc_ff_sub(u64 *out, const u64 *a, const u64 *b, size_t n)
{ for (size_t i = 0; i < n; i++) out[i] = ff_sub(a[i] % P, b[i] % P); }
void orc_ff_mul_prepared(u64 *out, const u64 *a, const u64 *b, size_t n)
{ for (size_t i = 0; i < n; i++) out[i] = ff_mul_prepared(a[i], b[i]); }
void orc_ff_prepare_for_mul(u64 *out, const u64 *a, size_t n)
{ for (size_t i = 0; i < n; i++) out[i] = ff_prepare_for_mul(a[i]); }
/* x * 2^s mod p (arithmetic.mako:465-1045 `lsh`, s < 192) */
void orc_ff_lsh(u64 *out, const u64 *a, const u32 *s, size_t n)
{ for (size_t i = 0; i < n; i++) out[i] = ff_mul(a[i] % P, ff_pow(2, s[i])); }

/* ------------------------------------------------------------------ NTT ---------------------- */

static u64 g_psi_pow[NPOLY];       /* psi^j,              psi = ROOT_GEN^(2^32/2048): ntt.py:33-34 */
static u64 g_psi_inv_pow[NPOLY];   /* psi^-j * N^-1 ... kept separate below */
static u64 g_w_pow[NPOLY];         /* omega^j,            omega = ROOT_GEN^(2^32/1024): ntt_cpu.py:97-109 */
static u64 g_w_inv_pow[NPOLY];
static u64 g_n_inv;
static int g_tables_ready = 0;

static void init_tables(void)
{
    if (g_tables_ready) return;
    u64 psi = ff_pow(ROOT_GEN, (1ULL << 32) / (2 * NPOLY));
    u64 w = ff_mul(psi, psi);
    u64 psi_inv = ff_inv(psi), w_inv = ff_inv(w);
    g_psi_pow[0] = g_psi_inv_pow[0] = g_w_pow[0] = g_w_inv_pow[0] = 1;
    for (int i = 1; i < NPOLY; i++) {
        g_psi_pow[i] = ff_mul(g_psi_pow[i - 1], psi);
        g_psi_inv_pow[i] = ff_mul(g_psi_inv_pow[i - 1], psi_inv);
        g_w_pow[i] = ff_mul(g_w_pow[i - 1], w);
        g_w_inv_pow[i] = ff_mul(g_w_inv_pow[i - 1], w_inv);
    }
    g_n_inv = ff_inv(NPOLY);
    g_tables_ready = 1;
}
void orc_init(void) { init_tables(); }

#ifdef _OPENMP
#include <omp.h>
void orc_set_threads(int n) { if (n > 0) omp_set_num_threads(n); }
int orc_get_threads(void) { return omp_get_max_threads(); }
#else
void orc_set_threads(int n) { (void)n; }
int orc_get_threads(void) { return 1; }
#endif

/* returns 0 when the folded reduction agrees with the plain `% p` on edge values and n random pairs */
int orc_selftest(u64 seed, size_t n)
{
    static const u64 edge[] = {0, 1, 2, 0xffffffffULL, 0x100000000ULL, 0xffffffff00000000ULL,
                               P - 1, P - 2, 0x7fffffff80000000ULL, 0x7fffffff80000001ULL};
    const int ne = sizeof(edge) / sizeof(edge[0]);
    for (int i = 0; i < ne; i++)
        for (int j = 0; j < ne; j++)
            if (ff_mul(edge[i], edge[j]) != ff_mul_slow(edge[i], edge[j])) return 1;
    u64 s = seed | 1;
    for (size_t i = 0; i < n; i++) {
        s ^= s << 13; s ^= s >> 7; s ^= s << 17; u64 a = s % P;
        s ^= s << 13; s ^= s >> 7; s ^= s << 17; u64 b = s % P;
        if (ff_mul(a, b) != ff_mul_slow(a, b)) return 2;
    }
    return 0;
}

/* Cyclic length-1024 transform out[k] = sum_j a[j] w^(jk), natural order in and out.
 * Same result as fft_generic, ntt_cpu.py:145-185 (the butterfly network there is one particular
 * evaluation order of this sum; the field arithmetic is exact so the result is unique). */
static void ntt_cyclic(u64 *a, const u64 *wpow)
{
    /* bit-reversal permutation, then decimation-in-time butterflies */
    for (int i = 0, j = 0; i < NPOLY; i++) {
        if (j > i) { u64 t = a[i]; a[i] = a[j]; a[j] = t; }
        int m = NPOLY >> 1;
        while (m >= 1 && (j & m)) { j ^= m; m >>= 1; }
        j |= m;
    }
    for (int len = 2; len <= NPOLY; len <<= 1) {
        int half = len >> 1, step = NPOLY / len;
        for (int i = 0; i < NPOLY; i += len)
            for (int k = 0; k < half; k++) {
                u64 t = ff_mul(a[i + k + half], wpow[k * step]);
                u64 u = a[i + k];
                a[i + k] = ff_add(u, t);
                a[i + k + half] = ff_sub(u, t);
            }
    }
}

/* ntt_transform_ref(inverse=False), ntt.py:30-44: NTT_w(a_j * psi^j). `in` already in the field. */
static void ntt_forward_ff(u64 *out, const u64 *in)
{
    for (int j = 0; j < NPOLY; j++) out[j] = ff_mul(in[j], g_psi_pow[j]);
    ntt_cyclic(out, g_w_pow);
}

/* ntt_transform_ref(inverse=True), ntt.py:37-42: INTT_w(.) * N^-1 * psi^-j */
static void ntt_inverse_ff(u64 *out, const u64 *in)
{
    for (int j = 0; j < NPOLY; j++) out[j] = in[j];
    ntt_cyclic(out, g_w_inv_pow);
    for (int j = 0; j < NPOLY; j++) out[j] = ff_mul(ff_mul(out[j], g_n_inv), g_psi_inv_pow[j]);
}

/* forward_transform_ref, polynomial_transform_ntt.py:45-46 (i32_conversion=True) */
void orc_ntt_forward_i32(u64 *out, const i32 *in, size_t batch)
{
    init_tables();
#pragma omp parallel for schedule(static)
    for (size_t b = 0; b < batch; b++) {
        u64 tmp[NPOLY];
        for (int j = 0; j < NPOLY; j++) tmp[j] = ff_from_i32(in[b * NPOLY + j]);
        ntt_forward_ff(out + b * NPOLY, tmp);
    }
}
/* ntt_transform_ref(data) on uint64 data, ntt.py:30-44 (GaloisNumber reduces its input mod p) */
void orc_ntt_forward_u64(u64 *out, const u64 *in, size_t batch)
{
    init_tables();
#pragma omp parallel for schedule(static)
    for (size_t b = 0; b < batch; b++) {
        u64 tmp[NPOLY];
        for (int j = 0; j < NPOLY; j++) tmp[j] = in[b * NPOLY + j] % P;
        ntt_forward_ff(out + b * NPOLY, tmp);
    }
}
void orc_ntt_inverse_u64(u64 *out, const u64 *in, size_t batch)
{
    init_tables();
#pragma omp parallel for schedule(static)
    for (size_t b = 0; b < batch; b++) {
        u64 tmp[NPOLY];
        for (int j = 0; j < NPOLY; j++) tmp[j] = in[b * NPOLY + j] % P;
        ntt_inverse_ff(out + b * NPOLY, tmp);
    }
}
/* inverse_transform_ref, polynomial_transform_ntt.py:49-50 */
void orc_ntt_inverse_i32(i32 *out, const u64 *in, size_t batch)
{
    init_tables();
#pragma omp parallel for schedule(static)
    for (size_t b = 0; b < batch; b++) {
        u64 tmp[NPOLY], res[NPOLY];
        for (int j = 0; j < NPOLY; j++) tmp[j] = in[b * NPOLY + j] % P;
        ntt_inverse_ff(res, tmp);
        for (int j = 0; j < NPOLY; j++) out[b * NPOLY + j] = ff_to_i32(res[j]);
    }
}

/* ------------------------------------------------------------------ scalar helpers ----------- */

/* Torus32ToPhaseReference, numeric_functions_cpu.py:23-37 */
void orc_t32_to_phase(i32 *out, const i32 *in, size_t n, u32 mspace_size)
{
    u32 interv = (u32)((1ULL << 32) / mspace_size), half = interv / 2;
    for (size_t i = 0; i < n; i++) out[i] = (i32)(((u32)in[i] + half) / interv);
}

/* One polynomial of ShiftTorusPolynomialReference, polynomials_cpu.py:25-59.
 * res = X^power * src (power in [0, 2N]), optionally minus src.  res must not alias src. */
static void shift_poly_one(i32 *res, const i32 *src, int power, int minus_one)
{
    const int N = NPOLY;
    if (power < N) {
        for (int x = 0; x < power; x++) res[x] = (i32)(0u - (u32)src[x + N - power]);
        for (int x = power; x < N; x++) res[x] = src[x - power];
    } else {
        int q = power - N;
        for (int x = 0; x < q; x++) res[x] = src[x + N - q];
        for (int x = q; x < N; x++) res[x] = (i32)(0u - (u32)src[x - q]);
    }
    if (minus_one)
        for (int x = 0; x < N; x++) res[x] = (i32)((u32)res[x] - (u32)src[x]);
}

/* ShiftTorusPolynomialReference, polynomials_cpu.py:25-59.
 * result/source: (batch, polys, N); powers: (batch, powers_stride) read at [b*powers_stride+powers_idx]
 * (powers_view=True) or (batch,) with powers_stride=1, powers_idx=0. */
void orc_shift_torus_polynomial(i32 *result, const i32 *source, const i32 *powers,
                                size_t batch, size_t polys, size_t powers_stride, size_t powers_idx,
                                int minus_one, int invert_powers)
{
    for (size_t b = 0; b < batch; b++) {
        int power = powers[b * powers_stride + powers_idx];
        if (invert_powers) power = 2 * NPOLY - power;
        for (size_t q = 0; q < polys; q++)
            shift_poly_one(result + (b * polys + q) * NPOLY, source + (b * polys + q) * NPOLY,
                           power, minus_one);
    }
}

/* TLweNoiselessTrivialReference, tlwe_cpu.py:26-38: acc (B,k+1,N) = (0, mu) */
void orc_tlwe_noiseless_trivial(i32 *acc, const i32 *mu, size_t batch)
{
    for (size_t b = 0; b < batch; b++) {
        memset(acc + b * 2 * NPOLY, 0, sizeof(i32) * NPOLY * MASK_K);
        memcpy(acc + (b * 2 + 1) * NPOLY, mu + b * NPOLY, sizeof(i32) * NPOLY);
    }
}

/* TLweExtractLweSamplesReference, tlwe_cpu.py:41-60 */
void orc_tlwe_extract_lwe_samples(i32 *res_a, i32 *res_b, const i32 *acc, size_t batch)
{
    for (size_t b = 0; b < batch; b++) {
        const i32 *a0 = acc + b * 2 * NPOLY, *a1 = a0 + NPOLY;
        i32 *ra = res_a + b * NPOLY;
        ra[0] = a0[0];
        for (int x = 1; x < NPOLY; x++) ra[x] = (i32)(0u - (u32)a0[NPOLY - x]);
        res_b[b] = a1[0];
    }
}

/* tgsw_polynomial_decomp_trf_reference, tgsw_cpu.py:26-49; offset from TGswParams, tgsw.py:48-53 */
static inline void decompose_coeff(i32 c, i32 *d0, i32 *d1)
{
    const u32 offset = 0x80000000u + (1u << (31 - BS_LOG2_BASE));   /* 2^31 + 2^21 */
    i32 t = (i32)((u32)c + offset);
    *d0 = ((t >> (32 - 1 * BS_LOG2_BASE)) & 1023) - 512;
    *d1 = ((t >> (32 - 2 * BS_LOG2_BASE)) & 1023) - 512;
}
/* result (B, k+1, l, N) from sample (B, k+1, N) */
void orc_tgsw_decompose(i32 *result, const i32 *sample, size_t batch)
{
    for (size_t b = 0; b < batch; b++)
        for (int m = 0; m < 2; m++)
            for (int x = 0; x < NPOLY; x++) {
                i32 d0, d1;
                decompose_coeff(sample[(b * 2 + m) * NPOLY + x], &d0, &d1);
                result[((b * 2 + m) * 2 + 0) * NPOLY + x] = d0;
                result[((b * 2 + m) * 2 + 1) * NPOLY + x] = d1;
            }
}

/* tlwe_transformed_add_mul_to_trf_reference, tgsw_cpu.py:52-79:
 * res[b][mo][x] = sum_{mi,j} mul_prepared(tr[b][mi][j][x], bk[row][mi][j][mo][x]) */
static void mac_one(u64 *res /*2,N*/, const u64 *tr /*2,2,N*/, const u64 *bk_row /*2,2,2,N*/)
{
    for (int mo = 0; mo < 2; mo++)
        for (int x = 0; x < NPOLY; x++) {
            u64 acc = 0;
            for (int mi = 0; mi < 2; mi++)
                for (int j = 0; j < 2; j++)
                    acc = ff_add(acc, ff_mul_prepared(tr[(mi * 2 + j) * NPOLY + x],
                                                      bk_row[((mi * 2 + j) * 2 + mo) * NPOLY + x]));
            res[mo * NPOLY + x] = acc;
        }
}
void orc_tgsw_mac(u64 *res, const u64 *tr, const u64 *bk, size_t bk_row, size_t batch)
{
    const u64 *row = bk + bk_row * 8 * NPOLY;
#pragma omp parallel for schedule(static)
    for (size_t b = 0; b < batch; b++) mac_one(res + b * 2 * NPOLY, tr + b * 4 * NPOLY, row);
}

/* TGswTransformedExternalMulReference, tgsw_cpu.py:82-106: accum <- bk[row] (x) accum (overwrites) */
static void external_mul_one(i32 *accum /*2,N*/, const u64 *bk_row)
{
    u64 tr[4 * NPOLY], mac[2 * NPOLY], tmp[NPOLY], res[NPOLY];
    for (int m = 0; m < 2; m++) {
        u64 d0[NPOLY], d1[NPOLY];
        for (int x = 0; x < NPOLY; x++) {
            i32 a, b;
            decompose_coeff(accum[m * NPOLY + x], &a, &b);
            d0[x] = ff_from_i32(a);
            d1[x] = ff_from_i32(b);
        }
        ntt_forward_ff(tr + (m * 2 + 0) * NPOLY, d0);
        ntt_forward_ff(tr + (m * 2 + 1) * NPOLY, d1);
    }
    mac_one(mac, tr, bk_row);
    for (int mo = 0; mo < 2; mo++) {
        memcpy(tmp, mac + mo * NPOLY, sizeof(tmp));
        ntt_inverse_ff(res, tmp);
        for (int x = 0; x < NPOLY; x++) accum[mo * NPOLY + x] = ff_to_i32(res[x]);
    }
}
void orc_tgsw_external_mul(i32 *accum, const u64 *bk, size_t bk_row, size_t batch)
{
    init_tables();
    const u64 *row = bk + bk_row * 8 * NPOLY;
#pragma omp parallel for schedule(static)
    for (size_t b = 0; b < batch; b++) external_mul_one(accum + b * 2 * NPOLY, row);
}

/* The same three steps for any TLWE mask size k (k1 = k + 1 accumulator polynomials), decomposition length 2:
 * what `NuFHEParameters(tlwe_mask_size=2)` runs (tgsw_cpu.py:26-106 are written for general k).
 * decomposition: result (polys, 2, N) from sample (polys, N) */
void orc_tgsw_decompose_polys(i32 *result, const i32 *sample, size_t polys)
{
    for (size_t p = 0; p < polys; p++)
        for (int x = 0; x < NPOLY; x++)
            decompose_coeff(sample[p * NPOLY + x], &result[(p * 2 + 0) * NPOLY + x], &result[(p * 2 + 1) * NPOLY + x]);
}
/* res (B, k1, N) = sum_{mi,j} mul_prepared(tr (B, k1, 2, N), bk_row (k1, 2, k1, N)) */
static void mac_one_k(u64 *res, const u64 *tr, const u64 *bk_row, int k1)
{
    for (int mo = 0; mo < k1; mo++)
        for (int x = 0; x < NPOLY; x++) {
            u64 acc = 0;
            for (int mi = 0; mi < k1; mi++)
                for (int j = 0; j < 2; j++)
                    acc = ff_add(acc, ff_mul_prepared(tr[(mi * 2 + j) * NPOLY + x],
                                                      bk_row[((mi * 2 + j) * k1 + mo) * NPOLY + x]));
            res[mo * NPOLY + x] = acc;
        }
}
void orc_tgsw_mac_k(u64 *res, const u64 *tr, const u64 *bk_row, size_t batch, int k1)
{
#pragma omp parallel for schedule(static)
    for (size_t b = 0; b < batch; b++) mac_one_k(res + b * k1 * NPOLY, tr + b * k1 * 2 * NPOLY, bk_row, k1);
}
/* accum (B, k1, N) <- bk_row (x) accum */
void orc_tgsw_external_mul_k(i32 *accum, const u64 *bk_row, size_t batch, int k1)
{
    init_tables();
#pragma omp parallel for schedule(static)
    for (size_t b = 0; b < batch; b++) {
        i32 *acc = accum + b * k1 * NPOLY;
        u64 tr[8 * 2 * NPOLY] = {0}, mac[8 * NPOLY], d0[NPOLY], d1[NPOLY], res[NPOLY];   /* k1 <= 8 */
        for (int m = 0; m < k1; m++) {
            for (int x = 0; x < NPOLY; x++) {
                i32 a, c;
                decompose_coeff(acc[m * NPOLY + x], &a, &c);
                d0[x] = ff_from_i32(a);
                d1[x] = ff_from_i32(c);
            }
            ntt_forward_ff(tr + (m * 2 + 0) * NPOLY, d0);
            ntt_forward_ff(tr + (m * 2 + 1) * NPOLY, d1);
        }
        mac_one_k(mac, tr, bk_row, k1);
        for (int mo = 0; mo < k1; mo++) {
            memcpy(d0, mac + mo * NPOLY, sizeof(d0));
            ntt_inverse_ff(res, d0);
            for (int x = 0; x < NPOLY; x++) acc[mo * NPOLY + x] = ff_to_i32(res[x]);
        }
    }
}

/* mux_rotate, bootstrap.py:96-109: ACC <- ACC + BK_i (x) ((X^bara_i - 1) ACC), one ciphertext */
static void mux_rotate_one(i32 *acc /*2,N*/, const u64 *bk_row, int barai)
{
    i32 tmp[2 * NPOLY];
    shift_poly_one(tmp, acc, barai, 1);
    shift_poly_one(tmp + NPOLY, acc + NPOLY, barai, 1);
    external_mul_one(tmp, bk_row);
    for (int x = 0; x < 2 * NPOLY; x++) acc[x] = (i32)((u32)acc[x] + (u32)tmp[x]);  /* tlwe.py:173-175 */
}

/* blind_rotate, bootstrap.py:119-142, batch version on (B,2,N) accumulators; bara (B, n) */
void orc_blind_rotate(i32 *acc, const u64 *bk, const i32 *bara, size_t n, size_t batch)
{
    init_tables();
#pragma omp parallel for schedule(dynamic, 1)
    for (size_t b = 0; b < batch; b++)
        for (size_t i = 0; i < n; i++)
            mux_rotate_one(acc + b * 2 * NPOLY, bk + i * 8 * NPOLY, bara[b * n + i]);
}

/* The multi-bit blind rotation of nufhe_b200 (DESIGN.md section 14; the reference has no multi-bit key), built from the
 * restated steps above.  Key bits are taken two at a time; group g reads rows 3g, 3g+1, 3g+2 of bk (TGSW encryptions
 * of the indicators of the bit patterns p = 1, 2, 3, p = s_2g + 2 s_2g+1) and does
 *     ACC += sum_p (X^{k_p} - 1) (Dec(ACC) (x) BK_{g,p}),   k_1 = bara_2g, k_2 = bara_2g+1, k_3 = k_1 + k_2 mod 2N.
 * Every external product is the exact integer product reduced mod 2^32 (its coefficients stay far below p / 2), and
 * multiplication by X^k - 1 commutes with that reduction, so the result is exact.  acc (B,2,N); bara (B, n), n even. */
static void mux_rotate_mb_one(i32 *acc /*2,N*/, const u64 *bk_group /*3 rows*/, int k0, int k1)
{
    const int ks[3] = {k0, k1, (k0 + k1) % (2 * NPOLY)};
    i32 prod[2 * NPOLY], rot[2 * NPOLY];
    u32 sum[2 * NPOLY] = {0};
    for (int p = 0; p < 3; p++) {
        memcpy(prod, acc, sizeof(prod));
        external_mul_one(prod, bk_group + (size_t)p * 8 * NPOLY);
        shift_poly_one(rot, prod, ks[p], 1);
        shift_poly_one(rot + NPOLY, prod + NPOLY, ks[p], 1);
        for (int x = 0; x < 2 * NPOLY; x++) sum[x] += (u32)rot[x];
    }
    for (int x = 0; x < 2 * NPOLY; x++) acc[x] = (i32)((u32)acc[x] + sum[x]);
}

void orc_blind_rotate_mb(i32 *acc, const u64 *bk, const i32 *bara, size_t n, size_t batch)
{
    init_tables();
#pragma omp parallel for schedule(dynamic, 1)
    for (size_t b = 0; b < batch; b++)
        for (size_t g = 0; g < n / 2; g++)
            mux_rotate_mb_one(acc + b * 2 * NPOLY, bk + g * 3 * 8 * NPOLY, bara[b * n + 2 * g], bara[b * n + 2 * g + 1]);
}

/* LweKeyswitchReference, lwe_cpu.py:62-93.  ks_a (in, t, base, out), ks_b/ks_cv (in, t, base). */
void orc_lwe_keyswitch(i32 *res_a, i32 *res_b, float *res_cv,
                       const i32 *ks_a, const i32 *ks_b, const float *ks_cv,
                       const i32 *src_a, const i32 *src_b,
                       size_t batch, size_t input_size, size_t output_size,
                       int decomp_length, int log2_base)
{
    const int base = 1 << log2_base;
    const u32 prec_offset = 1u << (32 - (1 + log2_base * decomp_length));
#pragma omp parallel for schedule(static)
    for (size_t b = 0; b < batch; b++) {
        i32 *ra = res_a + b * output_size;
        u32 rb = (u32)src_b[b];
        float cvf = 0;     /* float32 running sum, as lwe_sub_to on a float32 array (lwe_cpu.py:90-93) */
        for (size_t i = 0; i < output_size; i++) ra[i] = 0;
        for (size_t l = 0; l < input_size; l++) {
            i32 tmp = (i32)((u32)src_a[b * input_size + l] + prec_offset);
            for (int j = 0; j < decomp_length; j++) {
                int x = (tmp >> (32 - (j + 1) * log2_base)) & (base - 1);
                /* row x = 0 of a well-formed key is zero (lwe_cpu.py:31-33) but the reference closure
                 * subtracts whatever is stored there, so we do too. */
                const i32 *row = ks_a + ((l * decomp_length + j) * base + x) * output_size;
                for (size_t i = 0; i < output_size; i++) ra[i] = (i32)((u32)ra[i] - (u32)row[i]);
                rb -= (u32)ks_b[(l * decomp_length + j) * base + x];
                cvf += ks_cv[(l * decomp_length + j) * base + x];
            }
        }
        res_b[b] = (i32)rb;
        res_cv[b] = cvf;
    }
}

/* ------------------------------------------------------------------ bootstrap & gates -------- */

/* bootstrap, bootstrap.py:206-229 -> blind_rotate_and_extract :154-196 (loop path).
 * in: (B, n) + (B,), out: extracted (B, N) + (B,) when ks_a == NULL, else key-switched (B, n). */
void orc_bootstrap(i32 *out_a, i32 *out_b, const i32 *in_a, const i32 *in_b,
                   const u64 *bk, const i32 *ks_a, const i32 *ks_b, const float *ks_cv,
                   i32 mu, size_t batch, size_t n, int ks_decomp_length, int ks_log2_base)
{
    init_tables();
    i32 *ext_a = ks_a ? malloc(sizeof(i32) * batch * NPOLY) : out_a;
    i32 *ext_b = ks_a ? malloc(sizeof(i32) * batch) : out_b;
#pragma omp parallel for schedule(dynamic, 1)
    for (size_t b = 0; b < batch; b++) {
        i32 bara[4096], barb, acc[2 * NPOLY], testvect[NPOLY];
        orc_t32_to_phase(&barb, in_b + b, 1, 2 * NPOLY);              /* bootstrap.py:220 */
        orc_t32_to_phase(bara, in_a + b * n, n, 2 * NPOLY);           /* bootstrap.py:221 */
        for (int x = 0; x < NPOLY; x++) testvect[x] = mu;             /* bootstrap.py:224 */
        memset(acc, 0, sizeof(i32) * NPOLY);                          /* bootstrap.py:181-182 */
        shift_poly_one(acc + NPOLY, testvect, 2 * NPOLY - barb, 0);   /* bootstrap.py:177-178 */
        for (size_t i = 0; i < n; i++) mux_rotate_one(acc, bk + i * 8 * NPOLY, bara[i]);
        orc_tlwe_extract_lwe_samples(ext_a + b * NPOLY, ext_b + b, acc, 1);   /* bootstrap.py:193 */
    }
    if (ks_a) {
        float *cv = malloc(sizeof(float) * batch);
        orc_lwe_keyswitch(out_a, out_b, cv, ks_a, ks_b, ks_cv, ext_a, ext_b, batch, NPOLY, n,
                          ks_decomp_length, ks_log2_base);            /* bootstrap.py:195-196 */
        free(cv); free(ext_a); free(ext_b);
    }
}

/* Linear prologue of the bootstrapped binary gates, gates.py:81-597:
 * t = (0, c) + sa*a + sb*b  (Torus32 wrap), one of the rows of SURVEY.md section 8 a1. */
void orc_lwe_affine2(i32 *t_a, i32 *t_b, const i32 *a_a, const i32 *a_b, const i32 *b_a, const i32 *b_b,
                     i32 c, i32 sa, i32 sb, size_t batch, size_t n)
{
    for (size_t i = 0; i < batch * n; i++)
        t_a[i] = (i32)((u32)sa * (u32)a_a[i] + (u32)sb * (u32)b_a[i]);
    for (size_t i = 0; i < batch; i++)
        t_b[i] = (i32)((u32)c + (u32)sa * (u32)a_b[i] + (u32)sb * (u32)b_b[i]);
}

/* ------------------------------------------------------------------ key generation ----------- */

/* transformed_space_mul_ref path of TLweEncryptZeroReference, tlwe_cpu.py:64-89:
 * res = a * b in Z[X]/(X^N+1) reduced with the field->int32 rule (b is (batch, N), a is one poly). */
void orc_poly_mul_i32(i32 *res, const i32 *a, const i32 *b, size_t batch)
{
    init_tables();
    u64 ta[NPOLY], fa[NPOLY];
    for (int j = 0; j < NPOLY; j++) fa[j] = ff_from_i32(a[j]);
    ntt_forward_ff(ta, fa);
#pragma omp parallel for schedule(static)
    for (size_t q = 0; q < batch; q++) {
        u64 fb[NPOLY], tb[NPOLY], r[NPOLY];
        for (int j = 0; j < NPOLY; j++) fb[j] = ff_from_i32(b[q * NPOLY + j]);
        ntt_forward_ff(tb, fb);
        for (int j = 0; j < NPOLY; j++) tb[j] = ff_mul(ta[j], tb[j]);
        ntt_inverse_ff(r, tb);
        for (int j = 0; j < NPOLY; j++) res[q * NPOLY + j] = ff_to_i32(r[j]);
    }
}

/* TLweTransformSamples, tlwe_gpu.py:199-236 = forward NTT then prepare_for_mul (arithmetic.py:172) */
void orc_bk_transform(u64 *out, const i32 *in, size_t npolys)
{
    orc_ntt_forward_i32(out, in, npolys);
    orc_ff_prepare_for_mul(out, out, npolys * NPOLY);
}

/* LweDecryptReference / LweEncryptReference dot product, lwe_cpu.py:22-23, 104-121 */
void orc_lwe_phase(i32 *res, const i32 *a, const i32 *b, const i32 *key, size_t batch, size_t n)
{
    for (size_t q = 0; q < batch; q++) {
        u32 s = 0;
        for (size_t i = 0; i < n; i++) s += (u32)a[q * n + i] * (u32)key[i];
        res[q] = (i32)((u32)b[q] - s);
    }
}
void orc_lwe_dot(i32 *res, const i32 *a, const i32 *key, size_t batch, size_t n)
{
    for (size_t q = 0; q < batch; q++) {
        u32 s = 0;
        for (size_t i = 0; i < n; i++) s += (u32)a[q * n + i] * (u32)key[i];
        res[q] = (i32)s;
    }
}
