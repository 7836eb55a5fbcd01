// kernels.cuh -- sm_90a kernels of the TFHE gate-bootstrapping hot path (SURVEY.md section 8 rows a3-a15).
//
// Work decomposition of the fused bootstrap: a CTA owns one or two ciphertexts whose accumulators and work
// polynomials live in shared memory; every CMux step is seven CTA-wide phases (br_phases.cuh) separated by
// __syncthreads, 16 field elements per thread and phase.  The kernel is persistent: at most one wave of CTAs, which
// pull (chain, chunk) work items from a FIFO of ready chains in global memory, so that any batch is spread over all SMs.
// The smallest batches take a second kernel that spreads ONE ciphertext over a cluster of two SMs (pair shape: the step
// divides along the two accumulator polynomials, one 8 KB exchange per step through distributed shared memory).
// The stand-alone transforms reuse the same phases behind cp.async-staged, 128-bit input / output.  The key switch is a
// TMA-fed producer / consumer pipeline.  Then the separate steps of the reference's multi-kernel bootstrap, and the
// key-generation kernels (LWE dot product, key-switch key).  The fused bootstrap kernels also have a programmable-bootstrap
// instantiation (template argument LUT): a test vector read from memory in the head, the phase rounded to multiples of
// 2^L, and 2^L samples extracted in the tail (lut_index.cuh).
//
// Reference counterparts: nufhe/blind_rotate.mako:18-226 (fused bootstrap), tgsw_gpu.py:110-169
// (external product), transform/computation.mako:18-143 (stand-alone transform), lwe_gpu.mako:59-118
// (key switch).  Nothing here is derived from those kernels' structure (128 threads/transform,
// 8*2*8*8 radix plan, 15 block barriers per step); see ntt_lane.cuh for the transform we use and DESIGN.md
// section 4 for the measurements behind each choice.
#pragma once
#include <cuda_runtime.h>
#include <type_traits>
#include "ntt_lane.cuh"
#include "br_phases.cuh"
#include "lut_index.cuh"
#include "chacha.cuh"
#include "pk_layout.cuh"
#include "pack_layout.cuh"
#include "tree_layout.cuh"
#include "mk_layout.cuh"
#include "mk_expand_layout.cuh"

namespace nb {

constexpr int LWE_N_MAX = 1024;          // upper bound on the LWE dimension n handled by the gate kernels

NB_D u32 smem_u32(const void *p) { return (u32)__cvta_generic_to_shared(p); }
NB_D void cp_async16(void *smem, const void *gmem)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem)), "l"(gmem) : "memory");
}
NB_D void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> NB_D void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// ---- stand-alone batched transforms (reference: transform/computation.mako `standalone_transform`) ---
// natural order in and out.  Same three passes as the fused bootstrap (br_phases.cuh), 4 polynomials per
// sweep of 256 threads, 2 persistent CTAs per SM.  The natural-order side never meets the arithmetic directly:
//   * the next sweep's input is fetched with cp.async (16 bytes per request) into a second staging buffer while the
//     current sweep computes, so no pass waits on global memory;
//   * a thread owns the natural-order pairs (2t, 2t+1) and (2t+512, 2t+513) of every polynomial: in the pass layout
//     those four elements sit in two 16-byte shared-memory words 8 rows apart (ntt_pair_position), so the u64 side is
//     moved with 128-bit shared AND 128-bit global accesses (512 contiguous bytes per warp), bank-conflict free;
//   * the int32 side is read from / written to global memory as 128-byte warp rows (x[64 j1 + j2], lanes = j2).
#ifndef NB_NTT_CTAS
#define NB_NTT_CTAS 3                      // resident CTAs per SM of the stand-alone transforms (3 measured faster than 2)
#endif
constexpr int NTT_CTAS = NB_NTT_CTAS;
constexpr int NTT_RAW_I32_BYTES = NTT_SWEEP_POLYS * NTT_N * (int)sizeof(i32);
constexpr int NTT_RAW_U64_BYTES = NTT_SWEEP_POLYS * NTT_N * (int)sizeof(u64);
// staging buffers per CTA: two (prefetch one sweep ahead) unless three CTAs of u64 input have to share the SM
NB_HDC int ntt_raw_buffers(int raw_bytes) { return (NTT_CTAS > 2 && raw_bytes > NTT_RAW_I32_BYTES) ? 1 : 2; }
NB_HDC size_t ntt_smem_bytes(int raw_bytes)
{
    return (size_t)NTT_SWEEP_POLYS * POLY_STRIDE * sizeof(u64) + NTT_N * sizeof(u64) + ntt_raw_buffers(raw_bytes) * (size_t)raw_bytes;
}

// shared-memory position (in u64) of natural element k = 2 t of a polynomial, t = threadIdx.x in [0, 256): the
// elements 2t+1, 2t+512 and 2t+513 are at +8 rows, +1 and +8 rows +1 (k1 = k % 16 is even, so brev4(k1 + 1) =
// brev4(k1) + 8; adding 512 to k sets the top bit of k2 >> 2, i.e. bit 0 of the stored column index)
NB_D int ntt_pair_position(int t)
{
    const int row = brev(2 * (t & 7), 4), u = brev((t >> 3) & 3, 2), i0 = brev(t >> 5, 4);
    return row * ROW_STRIDE + col_of(u, i0);
}
NB_D u64 ff_zero_if_p(u64 x) { return x == FF_P ? 0 : x; }       // [0, p] -> canonical

// stage one sweep (4 polynomials, clamped at the end of the batch) with 16-byte cp.async requests
template <int POLY_BYTES> NB_D void ntt_stage(unsigned char *raw, const unsigned char *in, size_t p0, size_t batch, int tid)
{
    constexpr int CHUNKS = POLY_BYTES / 16;
#pragma unroll
    for (int pl = 0; pl < NTT_SWEEP_POLYS; pl++) {
        const size_t p = min(p0 + pl, batch - 1);
        for (int c = tid; c < CHUNKS; c += NTT_SWEEP_THREADS)
            cp_async16(raw + pl * POLY_BYTES + c * 16, in + p * POLY_BYTES + (size_t)c * 16);
    }
}

template <bool IN_I32>
__global__ void __launch_bounds__(NTT_SWEEP_THREADS, NTT_CTAS) ntt_forward_kernel(const void *__restrict__ in, u64 *__restrict__ out,
                                                                            const u64 *__restrict__ twd_g, size_t batch)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    constexpr int POLY_BYTES = NTT_N * (IN_I32 ? 4 : 8), RAW_BYTES = NTT_SWEEP_POLYS * POLY_BYTES;
    u64 *w = reinterpret_cast<u64 *>(smem_raw);
    u64 *twd = w + NTT_SWEEP_POLYS * POLY_STRIDE;
    unsigned char *raw = reinterpret_cast<unsigned char *>(twd + NTT_N);
    const int tid = threadIdx.x;
    const size_t stride = (size_t)gridDim.x * NTT_SWEEP_POLYS;
    size_t p0 = (size_t)blockIdx.x * NTT_SWEEP_POLYS;
    if (p0 < batch) ntt_stage<POLY_BYTES>(raw, (const unsigned char *)in, p0, batch, tid);
    cp_async_commit();
    for (int i = tid; i < NTT_N; i += NTT_SWEEP_THREADS) twd[i] = twd_g[i];
    const int pos = ntt_pair_position(tid);
    constexpr int NBUF = ntt_raw_buffers(RAW_BYTES);
    int buf = 0;
    for (; p0 < batch; p0 += stride, buf ^= (NBUF - 1)) {
        if (NBUF == 2) {
            if (p0 + stride < batch) ntt_stage<POLY_BYTES>(raw + (buf ^ 1) * RAW_BYTES, (const unsigned char *)in, p0 + stride, batch, tid);
            cp_async_commit();
            cp_async_wait<1>();                   // everything but the group just committed has landed
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        {   // pass 1: thread = (poly, j2), reads x[64 j1 + j2] from the staging buffer
            const int pl = tid >> 6, j2 = tid & 63;
            const unsigned char *src = raw + buf * RAW_BYTES + pl * POLY_BYTES;
            if (IN_I32) {
                i32 x[16];
#pragma unroll
                for (int j1 = 0; j1 < 16; j1++) x[j1] = reinterpret_cast<const i32 *>(src)[64 * j1 + j2];
                phase_fwd1_i32(tid, x, w, twd);
            } else {
                u64 x[16];
#pragma unroll
                for (int j1 = 0; j1 < 16; j1++) x[j1] = ff_canon(reinterpret_cast<const u64 *>(src)[64 * j1 + j2]);
                phase_fwd1_generic(tid, x, w, twd);
            }
        }
        __syncthreads();
        { const int g = tid >> 6, x = tid & 63; phase_fwd2(x >> 4, x & 15, g, w); }
        __syncthreads();
        if (NBUF == 1 && p0 + stride < batch) {   // single staging buffer: refill it now that pass 1 has consumed it
            ntt_stage<POLY_BYTES>(raw, (const unsigned char *)in, p0 + stride, batch, tid);
            cp_async_commit();
        }
        { const int u = tid & 3, r = (tid >> 2) & 15, p = tid >> 6; phase_fwd3(p, r, u, w); }
        __syncthreads();
        // natural-order store: 16 bytes = elements (2t, 2t+1) and (2t+512, 2t+513) of each polynomial
#pragma unroll
        for (int pl = 0; pl < NTT_SWEEP_POLYS; pl++) {
            if (p0 + pl < batch) {
                u64 a0, a1, b0, b1;
                ld2(w + pl * POLY_STRIDE + pos, a0, a1);                       // k = 2t, 2t + 512
                ld2(w + pl * POLY_STRIDE + pos + 8 * ROW_STRIDE, b0, b1);      // k = 2t + 1, 2t + 513
                ulonglong2 *dst = reinterpret_cast<ulonglong2 *>(out + (p0 + pl) * NTT_N);
                dst[tid] = make_ulonglong2(ff_zero_if_p(a0), ff_zero_if_p(b0));
                dst[tid + 256] = make_ulonglong2(ff_zero_if_p(a1), ff_zero_if_p(b1));
            }
        }
        __syncthreads();
    }
    cp_async_wait<0>();
}

template <bool OUT_I32>
__global__ void __launch_bounds__(NTT_SWEEP_THREADS, NTT_CTAS) ntt_inverse_kernel(const u64 *__restrict__ in, void *__restrict__ out,
                                                                            const u64 *__restrict__ twd_g, size_t batch)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    constexpr int POLY_BYTES = NTT_N * 8, RAW_BYTES = NTT_SWEEP_POLYS * POLY_BYTES;
    u64 *w = reinterpret_cast<u64 *>(smem_raw);
    u64 *twd = w + NTT_SWEEP_POLYS * POLY_STRIDE;
    unsigned char *raw = reinterpret_cast<unsigned char *>(twd + NTT_N);
    const int tid = threadIdx.x;
    const size_t stride = (size_t)gridDim.x * NTT_SWEEP_POLYS;
    size_t p0 = (size_t)blockIdx.x * NTT_SWEEP_POLYS;
    if (p0 < batch) ntt_stage<POLY_BYTES>(raw, (const unsigned char *)in, p0, batch, tid);
    cp_async_commit();
    for (int i = tid; i < NTT_N; i += NTT_SWEEP_THREADS) twd[i] = twd_g[i];
    const int pos = ntt_pair_position(tid);
    constexpr int NBUF = ntt_raw_buffers(RAW_BYTES);
    int buf = 0;
    for (; p0 < batch; p0 += stride, buf ^= (NBUF - 1)) {
        if (NBUF == 2) {
            if (p0 + stride < batch) ntt_stage<POLY_BYTES>(raw + (buf ^ 1) * RAW_BYTES, (const unsigned char *)in, p0 + stride, batch, tid);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        // natural order -> pass layout (the mirror image of the forward kernel's store), canonicalising on the way
#pragma unroll
        for (int pl = 0; pl < NTT_SWEEP_POLYS; pl++) {
            const ulonglong2 *src = reinterpret_cast<const ulonglong2 *>(raw + buf * RAW_BYTES + pl * POLY_BYTES);
            const ulonglong2 lo = src[tid], hi = src[tid + 256];
            st2(w + pl * POLY_STRIDE + pos, ff_canon(lo.x), ff_canon(hi.x));
            st2(w + pl * POLY_STRIDE + pos + 8 * ROW_STRIDE, ff_canon(lo.y), ff_canon(hi.y));
        }
        __syncthreads();
        if (NBUF == 1 && p0 + stride < batch) {   // single staging buffer: refill it now that it has been consumed
            ntt_stage<POLY_BYTES>(raw, (const unsigned char *)in, p0 + stride, batch, tid);
            cp_async_commit();
        }
        { const int u = tid & 3, r = (tid >> 2) & 15, p = tid >> 6; phase_inv3(p, r, u, w); }
        __syncthreads();
        { const int g = tid >> 6, x = tid & 63; phase_inv2(x >> 4, x & 15, g, w); }
        __syncthreads();
        {
            const int pl = tid >> 6, j2 = tid & 63;
            if (OUT_I32) {
                i32 y[16];
                phase_inv1_i32(tid, y, w, twd);
                if (p0 + pl < batch) {
#pragma unroll
                    for (int j1 = 0; j1 < 16; j1++) ((i32 *)out)[(p0 + pl) * NTT_N + 64 * j1 + j2] = y[j1];
                }
            } else {
                u64 y[16];
                phase_inv1_generic(tid, y, w, twd);
                if (p0 + pl < batch) {
#pragma unroll
                    for (int j1 = 0; j1 < 16; j1++) ((u64 *)out)[(p0 + pl) * NTT_N + 64 * j1 + j2] = ff_zero_if_p(y[j1]);
                }
            }
        }
        __syncthreads();
    }
    cp_async_wait<0>();
}

// ---- element-wise field ops (unit tests of the arithmetic; key generation) ----------------------
enum FfOp { FF_OP_ADD = 0, FF_OP_SUB = 1, FF_OP_MUL = 2, FF_OP_MUL_PREPARED = 3, FF_OP_PREPARE = 4, FF_OP_LSH = 5,
            FF_OP_LSH_CONST = 6 };   // 6: the compile-time-shift code paths of the transforms, for unit tests

__global__ void ff_elementwise_kernel(int op, const u64 *__restrict__ a, const u64 *__restrict__ b,
                                      u64 *__restrict__ out, size_t n, size_t b_period)
{
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        u64 x = ff_canon(a[i]);
        u64 y = b ? b[b_period ? i % b_period : i] : 0;
        u64 r;
        switch (op) {
        case FF_OP_ADD: r = ff_add(x, ff_canon(y)); break;
        case FF_OP_SUB: r = ff_sub(x, ff_canon(y)); break;
        case FF_OP_MUL: r = ff_mul(x, ff_canon(y)); break;
        case FF_OP_MUL_PREPARED: r = ff_mul_prepared(x, ff_canon(y)); break;
        case FF_OP_PREPARE: r = ff_prepare_for_mul(x); break;
        case FF_OP_LSH_CONST: {
            const int sh = (int)(y % 192);
            r = x;
            static_for<0, 192>([&](auto S) { if (sh == decltype(S)::value) r = ff_shl<decltype(S)::value>(x); });
            break;
        }
        default: r = ff_shl_var(x, (int)(y % 192)); break;
        }
        out[i] = ff_canon(r);
    }
}

// ---- bootstrap-key layout ------------------------------------------------------------------------
// reference row (nufhe/blind_rotate.py:112): [mi][j][mo][k], values NTT(bk) * 2^64 (Montgomery form).
// internal row: [m = (mi*2+j)*2+mo][row * 64 + stored column] (br_phases.cuh), plain values, so that the
// MAC phase reads, per thread, one 16-byte pair from each of the 8 planes, coalesced across the CTA.
// One thread per (row, position): 8 plain planes + the 2 correction planes (br_phases.cuh: BK_PLANES).
__global__ void bk_prepare_kernel(const u64 *__restrict__ bk_ref, u64 *__restrict__ bk_int,
                                  const u64 *__restrict__ ones512, size_t rows)
{
    const size_t total = rows * NTT_N;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t row = i >> 10;
        const int pos = (int)(i & 1023);
        const int k = w_natural_index(pos >> 6, pos & 63);
        u64 sum[2] = {0, 0};
#pragma unroll
        for (int m = 0; m < 8; m++) {
            u64 x = ff_mul(ff_canon(bk_ref[row * 8 * NTT_N + m * NTT_N + k]), FF_RINV);
            bk_int[row * BK_ROW_U64 + m * NTT_N + pos] = x;
            sum[m & 1] = ff_add(sum[m & 1], x);
        }
        bk_int[row * BK_ROW_U64 + 8 * NTT_N + pos] = ff_mul(sum[0], ones512[k]);
        bk_int[row * BK_ROW_U64 + 9 * NTT_N + pos] = ff_mul(sum[1], ones512[k]);
    }
}

// ---- FP64 part of the engine key (br_phases.cuh: FP64 step) ----------------------------------------------------------
// plain[i] = the reference key value i out of Montgomery form (natural order): the input of the inverse transform that
// recovers the key polynomials' coefficients
__global__ void bk_plain_kernel(const u64 *__restrict__ bk_ref, u64 *__restrict__ plain, size_t n)
{
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        plain[i] = ff_mul(ff_canon(bk_ref[i]), FF_RINV);
}
// The key spectra of key polynomial m of a row, for a CTA of 64 threads: thread n0 holds the centred integer
// coefficients k[j] = coefficient 64 j + n0; they are split into 16-bit halves and both halves transformed with the
// passes of the bootstrap into `spec`, then stored to bk_int + row * row_u64 + row_offset (fft_key_pos).
NB_D void bk_spectra_transform(const long long (&k)[16], cplx (&spec)[2][FFT_SPEC_CPLX], const cplx *__restrict__ tab,
                               u64 *__restrict__ bk_int, size_t row, size_t row_u64, size_t row_offset, int m, int n0)
{
    {
        double lo[16], hi[16];
        fft_split_key(k, lo, hi);
        fft_fwd1(n0, lo, spec[0], tab);
        fft_fwd1(n0, hi, spec[1], tab);
    }
    __syncthreads();
    fft_fwd2(n0 & 7, (n0 >> 3) & 3, spec[n0 >> 5]);      // 2 x 32 tasks (h, n2, k1)
    __syncthreads();
    for (int t = n0; t < 2 * FFT_M / 4; t += 64) fft_fwd3(t & 127, spec[t >> 7]);
    __syncthreads();
    cplx *out = reinterpret_cast<cplx *>(bk_int + row * row_u64 + row_offset);
    for (int P = n0; P < FFT_M; P += 64)
        for (int h = 0; h < 2; h++) out[fft_key_pos(m * 2 + h, P & 127, P >> 7)] = spec[h][fft_pass3_x(fft_pass3_group(P & 127), P >> 7)];
}

// One CTA of 64 threads per key polynomial (blockIdx.x = row * 8 + m): its coefficients mod p (natural order) must be
// centred 32-bit integers, transformed by bk_spectra_transform.  A coefficient outside [-2^31, 2^31) sets
// *not_integral (the key then keeps the NTT step everywhere).
// The spectra of row r go to bk_int + r * row_u64 + row_offset: after the NTT planes of an engine key row
// (BK_ROW_U64, BK_NTT_U64), or alone (BK_FFT_U64, 0: a multi-bit key).
__global__ void __launch_bounds__(64) bk_spectra_kernel(const u64 *__restrict__ coef, u64 *__restrict__ bk_int,
                                                        const cplx *__restrict__ tab, int *__restrict__ not_integral,
                                                        size_t row_u64, size_t row_offset)
{
    __shared__ __align__(16) cplx spec[2][FFT_SPEC_CPLX];
    const size_t poly = blockIdx.x, row = poly >> 3;
    const int m = (int)(poly & 7), n0 = threadIdx.x;
    long long k[16];
    bool bad = false;
#pragma unroll
    for (int j = 0; j < 16; j++) {
        const u64 v = ff_canon(coef[poly * NTT_N + 64 * j + n0]);
        const u64 half = 1ull << 31;
        if (v < half) k[j] = (long long)v;
        else if (v >= FF_P - half) k[j] = -(long long)(FF_P - v);
        else { k[j] = 0; bad = true; }
    }
    if (bad) atomicOr(not_integral, 1);
    bk_spectra_transform(k, spec, tab, bk_int, row, row_u64, row_offset, m, n0);
}

// ---- multi-key expansion of compressed cloud keys (DESIGN.md section 19; index arithmetic in mk_expand_layout.cuh)
// One tenant of nb_mk_bk_expand: its seed, bootstrap-key bodies (n, k+1, l, N) int32 and slot (n engine key rows)
struct MkBkTenant {
    u32 seed[8];
    const i32 *body;
    u64 *slot;
};

// The FP64 part of every row of every listed slot, k = 1, l = 2, N = 1024: one CTA of 64 threads per key polynomial,
// blockIdx.x = (tenant * n + row) * 8 + m with m = (mi * 2 + j) * 2 + mo as in bk_spectra_kernel.  A mask polynomial
// (mo = 0) is 64 ChaCha blocks, one per thread, regrouped through shared memory (aliased onto the spectra, which are
// written only after the regrouped words are in registers); a body polynomial (mo = 1) is read from the bodies.  The
// coefficients are the int32 values decompress() feeds nb_bk_prepare, so the spectra are the ones it stores.  The
// NTT planes of the rows are not written.
__global__ void __launch_bounds__(64) mk_bk_expand_kernel(const MkBkTenant *__restrict__ tenants, u32 n,
                                                          const cplx *__restrict__ tab)
{
    __shared__ __align__(16) cplx spec[2][FFT_SPEC_CPLX];
    static_assert(MK_REGROUP_WORDS * sizeof(u32) <= sizeof(spec), "the regrouping buffer lives in the spectra");
    const u64 poly = blockIdx.x, row_all = poly >> 3;
    const u32 tenant = (u32)(row_all / n);
    const u64 row = row_all - (u64)tenant * n;
    const int m = (int)(poly & 7), n0 = threadIdx.x;
    const u32 mi = (u32)m >> 2, j = ((u32)m >> 1) & 1, mo = (u32)m & 1;
    const MkBkTenant &t = tenants[tenant];
    long long k[16];
    if (mo == 0) {
        u32 *buf = reinterpret_cast<u32 *>(&spec[0][0]);
        u32 seed[8], x[16];
#pragma unroll
        for (int i = 0; i < 8; i++) seed[i] = t.seed[i];
        chacha20_block(seed, (mk_bk_mask_word(row, mi, j, mo, 1, 2, NTT_N) >> 4) + n0, MK_NONCE_BK, x);
#pragma unroll
        for (int w = 0; w < 16; w++) buf[mk_regroup_slot(16 * n0 + w)] = x[w];
        __syncthreads();
#pragma unroll
        for (int jj = 0; jj < 16; jj++) k[jj] = (i32)buf[mk_regroup_slot(mk_spectra_coef(n0, jj))];
        __syncthreads();
    } else {
        const i32 *body = t.body + mk_bk_body_offset(row, mi, j, 1, 2, NTT_N);
#pragma unroll
        for (int jj = 0; jj < 16; jj++) k[jj] = body[mk_spectra_coef(n0, jj)];
    }
    bk_spectra_transform(k, spec, tab, t.slot, row, BK_ROW_U64, BK_NTT_U64, m, n0);
}

// One tenant of nb_mk_ks_expand
struct MkKsTenant {
    u32 seed[8];
    i32 *ks_a;
};

constexpr int MK_KS_THREADS = 256;

// ks_a (in, t, base, n) of tenant blockIdx.y: the `words` mask words of the stream (seed, nonce 2) into rows h >= 1
// (mk_ks_a_word), as seeded_uniform_kernel writes a stream: a lane per block, a warp's 32 blocks staged through shared
// memory so that each store instruction writes 32 consecutive stream words; then zeros into the `zero_rows` rows h = 0.
__global__ void __launch_bounds__(MK_KS_THREADS) mk_ks_expand_kernel(const MkKsTenant *__restrict__ tenants, u64 words,
                                                                     u64 zero_rows, u32 n, u32 base)
{
    __shared__ u32 stage[MK_KS_THREADS / 32][32 * 17];
    const int lane = threadIdx.x & 31;
    u32 *st = stage[threadIdx.x >> 5];
    const MkKsTenant &tt = tenants[blockIdx.y];
    i32 *out = tt.ks_a;
    u32 seed[8];
#pragma unroll
    for (int i = 0; i < 8; i++) seed[i] = tt.seed[i];
    const u64 blocks = (words + 15) >> 4;
    const u64 thread = (u64)blockIdx.x * blockDim.x + threadIdx.x, threads = (u64)gridDim.x * blockDim.x;
    for (u64 wb = (thread >> 5) * 32; wb < blocks; wb += (threads >> 5) * 32) {
        if (wb + lane < blocks) {
            u32 x[16];
            chacha20_block(seed, wb + lane, MK_NONCE_KS, x);
#pragma unroll
            for (int j = 0; j < 16; j++) st[lane * 17 + j] = x[j];
        }
        __syncwarp();
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const int idx = j * 32 + lane;
            const u64 w = wb * 16 + idx;
            if (w < words) out[mk_ks_a_word(w, n, base)] = (i32)st[(idx >> 4) * 17 + (idx & 15)];
        }
        __syncwarp();
    }
    for (u64 i = thread; i < zero_rows * n; i += threads) out[mk_ks_zero_word(i / n, i % n, n, base)] = 0;
}

// mod-switch to [0, 2N) (numeric_functions_gpu.py:55-71)
NB_HD i32 modswitch_2n(i32 x) { return (i32)(((u32)x + (1u << 20)) >> 21); }

// ---- fused bootstrap: CTA-wide phases over shared-memory-resident polynomials (br_phases.cuh) -----
// u64 per work polynomial: an NTT work polynomial, or a padded spectrum of the FP64 step
template <class Cfg> NB_HDC int br_poly_u64() { return Cfg::FFT ? FFT_SPEC_CPLX * 2 : POLY_STRIDE; }
template <class Cfg> constexpr size_t br_smem_bytes()
{
    return (size_t)Cfg::CT * 2 * NTT_N * sizeof(i32) + (size_t)Cfg::POLYS * br_poly_u64<Cfg>() * sizeof(u64) +
           (Cfg::TWD_GLOBAL ? 0 : 2 * NTT_N * sizeof(u64)) + 64 + (Cfg::STAGE_KEY ? BK_NTT_U64 * sizeof(u64) : 0);
}
constexpr size_t BR2_SMEM_BYTES = br_smem_bytes<BrDefault>();

struct BlindRotateArgs {
    // mode A (gate): x = c + s1 * in1 + s2 * in2 is formed on the fly (gates.py prologues), then
    //                bootstrap(mu, x) (bootstrap.py:206-229).  in2 may be null (s2 ignored).
    const i32 *in1_a, *in1_b, *in2_a, *in2_b;
    i32 c, s1, s2, mu;
    // optional second job over the same launch (gate_mux's two bootstraps, gates.py:638-655): ciphertexts
    // [job_batch, 2 job_batch) use these operands / signs instead; outputs are simply the next rows
    const i32 *j2_in1_a, *j2_in1_b, *j2_in2_a, *j2_in2_b;
    i32 j2_c, j2_s1, j2_s2;
    size_t job_batch;       // 0: single job
    // mode B (BlindRotate_gpu, blind_rotate.py:262-281): explicit accumulator (B,2,1024) and bara (B,n)
    const i32 *accum, *bara;
    const u64 *bk;          // internal layout, n rows
    const cplx *fft_tab;    // tables of the FP64 step (tables.h: FftTables)
    i32 *out_a, *out_b;     // extracted LWE samples (B,1024), (B,)
    i32 *accum_out;         // optional: final accumulators (B,2,1024)
    int n;                  // LWE dimension (500); n = 0 with `plain` = one external product
    int extract;            // write out_a/out_b
    int plain;              // 1: accum <- bk[0] (x) accum, no rotation (tgsw.py:165-172), n ignored
    size_t batch;
    // work queue (see blind_rotate_kernel): `chains` groups of Cfg::CT ciphertexts, each cut into `chunks` runs of
    // `steps_per_chunk` CMux steps.  sched == null: one chain per CTA, no queue (single wave).
    unsigned *sched;        // [0] = queue head, [1] = entries appended so far, [BR_SCHED_HEADER + t] = entry t of the ready queue
    i32 *state;             // accumulators parked between the chunks of a chain: (chains * CT, 2, 1024)
    unsigned chains, chunks;
    int steps_per_chunk;
    int sm_count, stagger_cycles;   // single-wave launches: the second CTA of every SM starts this much later
    // mode A with a test vector (the programmable bootstrap, the LUT instantiations of the kernels below):
    // ciphertext c starts from X^(2N - barb) * tv[c * tv_stride ..] instead of the constant mu; barb and every bara_i
    // are rounded to multiples of 2^log2_outputs, and samples are extracted at indices j = 0 .. 2^log2_outputs - 1
    // into rows c * 2^log2_outputs + j of out_a / out_b (lut_index.cuh)
    const i32 *tv;
    size_t tv_stride;       // 0: one test vector for the batch, NTT_N: one per ciphertext, 2 NTT_N: one GLWE per ciphertext
    int log2_outputs;
    // multi-key launches (the BrFftMk instantiation of blind_rotate_kernel; bk unused): the engine key of tenant t starts at mk_bk[t], and
    // ciphertext c of the batch belongs to tenant mk_tenant[c]
    const u64 *const *mk_bk;
    const unsigned *mk_tenant;
};
constexpr int BR_SCHED_HEADER = 32;      // the ticket counter has a 128-byte line of its own

struct Br2Smem {
    i32 *acc;      // [CT][2][1024]
    u64 *w;        // [16][POLY_STRIDE]
    u64 *twd_fwd;  // [16][64]
    u64 *twd_inv;
    int *rot;      // [2][CT], 64 bytes
    u64 *key;      // Cfg::STAGE_KEY: the NTT part of the key row of the current step, [BK_PLANES][1024]
};

template <class Cfg> NB_D Br2Smem br2_carve(unsigned char *raw)
{
    Br2Smem s;
    s.w = reinterpret_cast<u64 *>(raw);
    s.twd_fwd = s.w + Cfg::POLYS * br_poly_u64<Cfg>();
    s.twd_inv = s.twd_fwd + (Cfg::TWD_GLOBAL ? 0 : NTT_N);
    s.acc = reinterpret_cast<i32 *>(s.twd_inv + (Cfg::TWD_GLOBAL ? 0 : NTT_N));
    s.rot = reinterpret_cast<int *>(s.acc + Cfg::CT * 2 * NTT_N);
    s.key = reinterpret_cast<u64 *>(reinterpret_cast<unsigned char *>(s.rot) + 64);
    return s;
}

// rotation amount of ciphertext c at step i
NB_D int br2_rotation(const BlindRotateArgs &p, size_t c, int i)
{
    if (p.bara) return p.bara[c * p.n + i];
    if (p.job_batch && c >= p.job_batch) {
        const size_t d = c - p.job_batch;
        u32 xa = (u32)p.j2_s1 * (u32)p.j2_in1_a[d * p.n + i] + (p.j2_in2_a ? (u32)p.j2_s2 * (u32)p.j2_in2_a[d * p.n + i] : 0u);
        return modswitch_2n((i32)xa);
    }
    // Torus32 arithmetic wraps by design (XOR / XNOR use s = +-2): unsigned, like lwe_affine_kernel
    u32 xa = (u32)p.s1 * (u32)p.in1_a[c * p.n + i] + (p.in2_a ? (u32)p.s2 * (u32)p.in2_a[c * p.n + i] : 0u);
    return modswitch_2n((i32)xa);
}

// coefficient x of polynomial mi of ciphertext c's accumulator before the first step
NB_D i32 br2_initial_acc(const BlindRotateArgs &p, size_t c, int mi, int x)
{
    if (p.accum) return p.accum[(c * 2 + mi) * NTT_N + x];
    if (mi == 0) return 0;
    // ACC = (0, X^(2N - barb) * [mu, ..., mu])   (bootstrap.py:177-182, 224)
    u32 xb;
    if (p.job_batch && c >= p.job_batch) {
        const size_t d = c - p.job_batch;
        xb = (u32)p.j2_c + (u32)p.j2_s1 * (u32)p.j2_in1_b[d] + (p.j2_in2_b ? (u32)p.j2_s2 * (u32)p.j2_in2_b[d] : 0u);
    } else {
        xb = (u32)p.c + (u32)p.s1 * (u32)p.in1_b[c] + (p.in2_b ? (u32)p.s2 * (u32)p.in2_b[c] : 0u);
    }
    const int q = 2 * NTT_N - modswitch_2n((i32)xb);
    if (q < NTT_N) return x < q ? (i32)(0u - (u32)p.mu) : p.mu;
    return x < q - NTT_N ? p.mu : (i32)(0u - (u32)p.mu);
}

// The same two for the programmable bootstrap (single job, no explicit accumulator): rounded mod-switch, test vector
NB_D int lut_rotation(const BlindRotateArgs &p, size_t c, int i)
{
    u32 xa = (u32)p.s1 * (u32)p.in1_a[c * p.n + i] + (p.in2_a ? (u32)p.s2 * (u32)p.in2_a[c * p.n + i] : 0u);
    return modswitch_lut((i32)xa, p.log2_outputs);
}

// tv_stride 2N: one GLWE test vector (mask, body) per ciphertext (nb_bootstrap_glwe_lut_extract), whose mask
// polynomial starts the accumulator's mask instead of 0
NB_D i32 lut_initial_acc(const BlindRotateArgs &p, size_t c, int mi, int x)
{
    const bool glwe = p.tv_stride == 2 * NTT_N;
    if (mi == 0 && !glwe) return 0;
    const u32 xb = (u32)p.c + (u32)p.s1 * (u32)p.in1_b[c] + (p.in2_b ? (u32)p.s2 * (u32)p.in2_b[c] : 0u);
    return lut_head_coef(p.tv + c * p.tv_stride + (glwe ? mi * NTT_N : 0), modswitch_lut((i32)xb, p.log2_outputs), x);
}

template <bool LUT> NB_D int br_rotation(const BlindRotateArgs &p, size_t c, int i)
{
    if constexpr (LUT) return lut_rotation(p, c, i);
    else return br2_rotation(p, c, i);
}

template <bool LUT> NB_D i32 br_initial_acc(const BlindRotateArgs &p, size_t c, int mi, int x)
{
    if constexpr (LUT) return lut_initial_acc(p, c, mi, x);
    else return br2_initial_acc(p, c, mi, x);
}

// 16-byte cp.async requests for one key row, spread over `nthreads` threads (t = 0 .. nthreads - 1); one commit group
NB_D void br2_stage_key(u64 *key, const u64 *__restrict__ bk_row, int t, int nthreads)
{
    for (int x = t; x < BK_NTT_U64 / 2; x += nthreads) cp_async16(key + 2 * x, bk_row + 2 * x);
    cp_async_commit();
}

// next_bk_row (Cfg::STAGE_KEY): the key row of the following step, or null
template <bool ROTATE, class Cfg>
NB_D void br2_step(const Br2Smem &s, const u64 *__restrict__ bk_row, const int *rot, int tid, const u64 *__restrict__ next_bk_row = nullptr)
{
    // forward transforms of the digit polynomials (CT ciphertexts x 2 polynomials x 2 digits)
    if constexpr (Cfg::SPLIT_FWD) {
        // two threads (of different warps) per task, 8 outputs each; tasks mapped as in the 256-thread shape
        using Tasks = BrCfg<Cfg::CT, 256 * Cfg::CT>;
        int h, t;
        map_split_fwd<Cfg>(tid, h, t);
        if (h) phase_fwd1_split<ROTATE, 1>(t, s.acc, s.w, s.twd_fwd, rot); else phase_fwd1_split<ROTATE, 0>(t, s.acc, s.w, s.twd_fwd, rot);
        __syncthreads();
        { int p, r, g; map_fwd2<Tasks>(t, 0, p, r, g); if (h) phase_fwd2_split<1>(p, r, g, s.w); else phase_fwd2_split<0>(p, r, g, s.w); }
        __syncthreads();
        {
            int p, r, u;
            u64 v[16];
            map_fwd3<Tasks>(t, 0, p, r, u);
            phase_fwd3_split_load(p, r, u, s.w, v);
            __syncthreads();                               // in place: all loads before any store
            if (h) phase_fwd3_split_finish<1>(p, r, u, s.w, v); else phase_fwd3_split_finish<0>(p, r, u, s.w, v);
        }
        __syncthreads();
    } else {
        if constexpr (Cfg::FWD1_BOTH_DIGITS) {
            phase_fwd1_both_digits<ROTATE>(tid, s.acc, s.w, s.twd_fwd, rot);
        } else {
#pragma unroll 1
            for (int it = 0; it < Cfg::FWD_SWEEPS; it++) phase_fwd1<ROTATE>(it * Cfg::THREADS + tid, s.acc, s.w, s.twd_fwd, rot);
        }
        __syncthreads();
#pragma unroll 1
        for (int it = 0; it < Cfg::FWD_SWEEPS; it++) { int p, r, g; map_fwd2<Cfg>(tid, it, p, r, g); phase_fwd2(p, r, g, s.w); }
        __syncthreads();
#pragma unroll 1
        for (int it = 0; it < Cfg::FWD_SWEEPS; it++) { int p, r, u; map_fwd3<Cfg>(tid, it, p, r, u); phase_fwd3(p, r, u, s.w); }
        __syncthreads();
    }
    // multiply-accumulate with the key row (tgsw_gpu.py:58-107); each key element is fetched once per CTA
    if constexpr (Cfg::STAGE_KEY) phase_mac<Cfg, true>(tid, s.w, s.key);
    else phase_mac<Cfg>(tid, s.w, bk_row);
    __syncthreads();
    // inverse transforms of the output polynomials
    if constexpr (Cfg::SPLIT_INV) {
        // twice as many threads as tasks: two threads (of different warps) per task, 8 elements each, parked values
        // exchanged through the dead work polynomials (br_phases.cuh: split inverse phases); two more barriers
        int h, t;
        // threads beyond twice the task count (the upper half of the wide2 CTA, whole warps) have no inverse work: they
        // go straight to the barrier that ends the step, and the working warps synchronise among themselves on a
        // named barrier
        if (map_split<Cfg>(tid, h, t)) {
            constexpr int WORKERS = 2 * Cfg::INV_TASKS;
            auto sync_workers = [] {
                if constexpr (WORKERS == Cfg::THREADS) __syncthreads();
                else asm volatile("bar.sync 1, %0;" ::"n"(WORKERS) : "memory");
            };
            { int p, r, u; map_inv3<Cfg>(t, p, r, u); if (h) phase_inv3_split_a<1>(p, r, u, s.w); else phase_inv3_split_a<0>(p, r, u, s.w); }
            sync_workers();
            { int p, r, u; map_inv3<Cfg>(t, p, r, u); if (h) phase_inv3_split_b<1>(p, r, u, s.w); else phase_inv3_split_b<0>(p, r, u, s.w); }
            sync_workers();
            { int p, r, g; map_inv2_split<Cfg>(t, p, r, g); if (h) phase_inv2_split<1>(p, r, g, s.w); else phase_inv2_split<0>(p, r, g, s.w); }
            sync_workers();
            if (h) phase_inv1_split_a<1>(t, s.w, s.twd_inv); else phase_inv1_split_a<0>(t, s.w, s.twd_inv);
            sync_workers();
            if (h) phase_inv1_split_b<ROTATE, 1>(t, s.acc, s.w); else phase_inv1_split_b<ROTATE, 0>(t, s.acc, s.w);
        } else if constexpr (Cfg::STAGE_KEY) {
            if (next_bk_row) {
                br2_stage_key(s.key, next_bk_row, tid - 2 * Cfg::INV_TASKS, Cfg::THREADS - 2 * Cfg::INV_TASKS);
                cp_async_wait<0>();                            // landed before this thread reaches the barrier that ends the step
            }
        }
    } else {
        // (threads beyond Cfg::INV_TASKS idle: whole warps)
        { int p, r, u; if (map_inv3<Cfg>(tid, p, r, u)) phase_inv3(p, r, u, s.w); }
        __syncthreads();
        { int p, r, g; if (map_inv2<Cfg>(tid, p, r, g)) phase_inv2(p, r, g, s.w); }
        __syncthreads();
        if (tid < Cfg::INV_TASKS) phase_inv1<ROTATE>(tid, s.acc, s.w, s.twd_inv);
    }
}

// The thread index, read again (volatile, so not hoisted out of the step loop): every address of the FP64 step's phases
// is a per-thread base plus constants, and without this the compiler keeps all five phases' bases live across the
// whole loop -- about 70 bytes more spill at 128 registers.
NB_D int fft_step_tid()
{
    int t;
    asm volatile("mov.u32 %0, %%tid.x;" : "=r"(t));
    return t;
}

// The FP64 step (br_phases.cuh: FP64 step): five barrier-separated phases on spectra of 512 complex doubles, one task
// per thread in each; bk_row: the whole engine key row (its FP64 part is read).
// MB: one group of a multi-bit key (br_phases.cuh: fft_phase_mac_mb): bk_row = the group's 3 rows of spectra, rot = the
// group's two rotation amounts per ciphertext; fwd1 decomposes ACC itself and inv1 adds to it.
template <bool ROTATE, class Cfg, bool MB = false>
NB_D void br_fft_step(const Br2Smem &s, const u64 *__restrict__ bk_row, const int *rot, int /* tid */, const cplx *__restrict__ tab)
{
    static_assert(Cfg::CT == FFT_CT && Cfg::THREADS == 256, "the FP64 step's thread maps (fft_layout.cuh)");
    static_assert(!MB || ROTATE, "a multi-bit group always accumulates");
    cplx *spec = reinterpret_cast<cplx *>(s.w);
    int tid = fft_step_tid();
    fft_phase_fwd1<ROTATE && !MB>(tid, s.acc, spec, tab, rot);   // (ct, mi, n0), both digits
    __syncthreads();
    tid = fft_step_tid();
    fft_phase_fwd2(tid, spec);                              // (ct, n2, s, k1): DFT16, W64 twiddles
    __syncthreads();
    tid = fft_step_tid();
    if constexpr (MB) fft_phase_mac_mb(tid, spec, reinterpret_cast<const cplx *>(bk_row), tab, rot);   // (j, ct): DFT4, 3-row MAC, inverse DFT4
    else fft_phase_mac(tid, spec, reinterpret_cast<const cplx *>(bk_row + BK_NTT_U64));   // (j, ct): DFT4, MAC, inverse DFT4
    __syncthreads();
    tid = fft_step_tid();
    fft_phase_inv2(tid, spec);                              // (ct, n2, s, k1)
    __syncthreads();
    tid = fft_step_tid();
    fft_phase_inv1<ROTATE>(tid, s.acc, spec, tab);                // (ct, mo, n0), both key halves
}

NB_D unsigned ld_acquire_u32(const unsigned *p)
{
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
NB_D void st_release_u32(unsigned *p, unsigned v)
{
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// steps of a chain: p.n, or p.n / 2 groups of a multi-bit key (read where used, so that the other kernels keep their code)
template <bool MB> NB_D int br_chain_steps(const BlindRotateArgs &p)
{
    if constexpr (MB) return p.n / 2;
    else return p.n;
}

// The kernel is persistent: the grid is at most one wave of resident CTAs (Cfg::CTAS_PER_SM per SM) and every CTA
// pulls work items from a queue until none are left.  A work item is one CHUNK of one CHAIN: a chain is the whole
// blind rotation of Cfg::CT ciphertexts, a chunk `steps_per_chunk` consecutive CMux steps of it.  Cutting chains into
// chunks time-slices a batch that is not a multiple of the wave size over all SMs instead of leaving a partial last
// wave: 1024 ciphertexts take 1.73 wave-times instead of 2 (the host picks the chunk count, capi.cu: pick_chunks).
// Between chunks the accumulators (8 KB per ciphertext) are parked in global memory.
// The queue is a FIFO of READY chains in global memory: entry t (t = 0 .. chains * chunks - 1) holds 1 + chain +
// chains * chunk; the host memset leaves every entry 0 = "not written yet" and the kernel treats entries t < chains as
// the initial state (chain t, chunk 0).  A CTA takes the next entry with an atomic increment of the head and waits for
// that entry to be written; when it finishes a chunk that is not the chain's last, it parks the accumulators and
// appends the chain's next chunk at the tail (release).  Whoever pops it (acquire) finds the accumulators.  An entry
// a CTA waits for is always produced by a chunk that is running on another resident CTA, so the wait cannot deadlock,
// and a ready chain never waits behind an unready one -- with in-order tickets and per-chain progress counters, which
// this replaces, a launch with slightly more chains than CTAs lost time to such head-of-line waits.
// LUT: the programmable bootstrap (BlindRotateArgs::tv); its own instantiation, so that the gate kernels keep their code.
// MB: a multi-bit key (BrFft only): a chain is p.n / 2 groups of two key bits instead of p.n steps, p.bk holds 3 rows of
// BK_FFT_U64 per group, and s.rot holds both rotation amounts of the group per ciphertext ([parity][CT][2]).
// Cfg = BrFftMk: the multi-key instantiation -- ciphertexts under different keys (BlindRotateArgs::mk_bk).  Chains are
// consecutive pairs of the batch as always, so the two slots of a CTA may belong to two tenants.  Only pass 3 of the
// FP64 step reads the key, and fft_phase_mac serves slot tid & 1 from the pointer its thread passes (as
// index_lookup_kernel does), so each thread passes the key of its own slot's tenant, looked up again for every work item.
template <class Cfg, bool LUT = false, bool MB = false>
__global__ void __launch_bounds__(Cfg::THREADS, Cfg::CTAS_PER_SM) blind_rotate_kernel(BlindRotateArgs p, const u64 *__restrict__ twd_fwd_g,
                                                                       const u64 *__restrict__ twd_inv_g)
{
    constexpr bool MK = std::is_same<Cfg, BrFftMk>::value;
    static_assert(!MB || Cfg::FFT, "multi-bit keys run the FP64 step");
    static_assert(!MK || !MB, "multi-key launches take standard keys");
    extern __shared__ __align__(16) unsigned char smem_raw[];
    Br2Smem s = br2_carve<Cfg>(smem_raw);
    __shared__ unsigned s_item, s_entry;
    const int tid = threadIdx.x;
    if (Cfg::FFT) {
        // the FP64 step reads its tables through the L1 (p.fft_tab)
    } else if (Cfg::TWD_GLOBAL) {
        s.twd_fwd = const_cast<u64 *>(twd_fwd_g); s.twd_inv = const_cast<u64 *>(twd_inv_g);
    } else {
        for (int i = tid; i < NTT_N; i += Cfg::THREADS) { s.twd_fwd[i] = twd_fwd_g[i]; s.twd_inv[i] = twd_inv_g[i]; }
    }
    const unsigned total = p.chains * p.chunks;
    constexpr int ACC_WORDS = Cfg::CT * 2 * NTT_N;
    // Two CTAs share an SM.  In a single-wave launch they would march through the phases in lock step (the MAC is
    // multiplier-bound and stalls both integer pipes, the transform passes are adder-bound); started half a step apart
    // they fill each other's gaps -- what multi-wave launches drift into by themselves.
    if (Cfg::CTAS_PER_SM > 1 && !p.sched && p.stagger_cycles > 0 && blockIdx.x >= (unsigned)p.sm_count) {
        if (tid == 0) {
            const long long t0 = clock64();
            while (clock64() - t0 < p.stagger_cycles) { }
        }
        __syncthreads();
    }

    for (unsigned item = blockIdx.x;; ) {
        if (p.sched) {
            __syncthreads();                                   // everyone is done with the previous item
            if (tid == 0) s_item = atomicAdd(p.sched, 1u);
            __syncthreads();
            item = s_item;
        }
        if (item >= total) break;
        unsigned chunk = 0, chain = item;
        if (p.sched && item >= p.chains) {
            // entries beyond the initial ones are appended by the CTAs that finish chunks
            if (tid == 0) {
                unsigned e;
                while ((e = ld_acquire_u32(p.sched + BR_SCHED_HEADER + item)) == 0) __nanosleep(100);
                s_entry = e - 1;
            }
            __syncthreads();
            const unsigned e = s_entry;
            chunk = e / p.chains; chain = e - chunk * p.chains;
        }
        const size_t ct0 = (size_t)chain * Cfg::CT;
        // ciphertext slots beyond the batch replay the last ciphertext and store nothing
        auto ct_of = [&](int slot) { size_t c = ct0 + slot; return c < p.batch ? c : p.batch - 1; };
        const int step0 = (int)chunk * p.steps_per_chunk;
        const int step1 = p.plain ? 1 : min(br_chain_steps<MB>(p), step0 + p.steps_per_chunk);

        if (chunk == 0) {
            // accumulator initialisation: CT x 2 polynomials x 1024 coefficients
            for (int e = tid; e < ACC_WORDS; e += Cfg::THREADS) {
                const int slot = e >> 11, mi = (e >> 10) & 1, x = e & (NTT_N - 1);
                s.acc[e] = br_initial_acc<LUT>(p, ct_of(slot), mi, x);
            }
        } else {
            // resume a parked chain: its queue entry was published after the accumulators (release / acquire above)
            const int4 *src = reinterpret_cast<const int4 *>(p.state + (size_t)chain * ACC_WORDS);
            for (int e = tid; e < ACC_WORDS / 4; e += Cfg::THREADS) reinterpret_cast<int4 *>(s.acc)[e] = __ldcg(src + e);
        }

        if constexpr (Cfg::STAGE_KEY) {
            // first key row of this item (the rows after it are staged inside the steps)
            br2_stage_key(s.key, p.bk + (size_t)(p.plain ? 0 : step0) * BK_ROW_U64, tid, Cfg::THREADS);
            cp_async_wait<0>();
        }
        if (!MB && p.plain) {          // (never with a multi-bit key: capi.cu rejects it)
            __syncthreads();
            if constexpr (Cfg::FFT) br_fft_step<false, Cfg>(s, p.bk, s.rot, tid, p.fft_tab);
            else br2_step<false, Cfg>(s, p.bk, s.rot, tid);
            __syncthreads();
        } else if constexpr (MB) {
            // thread t < 2 CT loads bit t & 1 of the group for ciphertext slot t >> 1
            if (tid < 2 * Cfg::CT) s.rot[(step0 & 1) * 2 * Cfg::CT + tid] = br_rotation<LUT>(p, ct_of(tid >> 1), 2 * step0 + (tid & 1));
            __syncthreads();
            for (int i = step0; i < step1; i++) {
                int next = 0;
                if (tid < 2 * Cfg::CT && i + 1 < step1) next = br_rotation<LUT>(p, ct_of(tid >> 1), 2 * (i + 1) + (tid & 1));
                br_fft_step<true, Cfg, true>(s, p.bk + (size_t)i * 3 * BK_FFT_U64, s.rot + (i & 1) * 2 * Cfg::CT, tid, p.fft_tab);
                if (tid < 2 * Cfg::CT) s.rot[((i + 1) & 1) * 2 * Cfg::CT + tid] = next;
                __syncthreads();
            }
        } else {
            const u64 *mk_bk = nullptr;       // MK: the key of this thread's pass-3 slot
            if constexpr (MK) mk_bk = p.mk_bk[p.mk_tenant[ct_of(tid & 1)]];
            if (tid < Cfg::CT) s.rot[(step0 & 1) * Cfg::CT + tid] = br_rotation<LUT>(p, ct_of(tid), step0);
            __syncthreads();
            for (int i = step0; i < step1; i++) {
                int next = 0;
                if (tid < Cfg::CT && i + 1 < step1) next = br_rotation<LUT>(p, ct_of(tid), i + 1);
                if constexpr (MK)
                    br_fft_step<true, Cfg>(s, mk_bk + (size_t)i * BK_ROW_U64, s.rot + (i & 1) * Cfg::CT, tid, p.fft_tab);
                else if constexpr (Cfg::FFT)
                    br_fft_step<true, Cfg>(s, p.bk + (size_t)i * BK_ROW_U64, s.rot + (i & 1) * Cfg::CT, tid, p.fft_tab);
                else
                    br2_step<true, Cfg>(s, p.bk + (size_t)i * BK_ROW_U64, s.rot + (i & 1) * Cfg::CT, tid,
                                        i + 1 < step1 ? p.bk + (size_t)(i + 1) * BK_ROW_U64 : nullptr);
                if (tid < Cfg::CT) s.rot[((i + 1) & 1) * Cfg::CT + tid] = next;
                __syncthreads();
            }
        }

        if (!p.plain && step1 < br_chain_steps<MB>(p)) {
            // park the accumulators and publish the chain's progress
            int4 *dst = reinterpret_cast<int4 *>(p.state + (size_t)chain * ACC_WORDS);
            for (int e = tid; e < ACC_WORDS / 4; e += Cfg::THREADS) __stcg(dst + e, reinterpret_cast<const int4 *>(s.acc)[e]);
            __threadfence();
            __syncthreads();
            if (tid == 0) {
                const unsigned slot = p.chains + atomicAdd(p.sched + 1, 1u);   // appended entries follow the initial ones
                st_release_u32(p.sched + BR_SCHED_HEADER + slot, 1u + chain + p.chains * (chunk + 1));
            }
        } else if constexpr (LUT) {
            // samples j = 0 .. 2^L - 1 of every ciphertext, into rows c * 2^L + j
            const int L = p.log2_outputs;
            for (int e = tid; e < (Cfg::CT * NTT_N) << L; e += Cfg::THREADS) {
                const int slot = e >> (10 + L), j = (e >> 10) & ((1 << L) - 1), x = e & (NTT_N - 1);
                const size_t c = ct0 + slot;
                if (c >= p.batch) continue;
                const i32 *a0 = s.acc + slot * 2 * NTT_N;
                const size_t row = (c << L) + j;
                p.out_a[row * NTT_N + x] = lut_tail_a(a0, j, x);
                if (x == 0) p.out_b[row] = a0[NTT_N + j];
            }
        } else {
            for (int e = tid; e < ACC_WORDS; e += Cfg::THREADS) {
                const int slot = e >> 11, mi = (e >> 10) & 1, x = e & (NTT_N - 1);
                const size_t c = ct0 + slot;
                if (c >= p.batch) continue;
                if (p.accum_out) p.accum_out[(c * 2 + mi) * NTT_N + x] = s.acc[e];
                if (p.extract) {
                    // sample extraction (tlwe_gpu.mako:63-82; blind_rotate.mako:213-224)
                    const i32 *a0 = s.acc + slot * 2 * NTT_N;
                    if (mi == 0) p.out_a[c * NTT_N + x] = x == 0 ? a0[0] : (i32)(0u - (u32)a0[NTT_N - x]);
                    else if (x == 0) p.out_b[c] = a0[NTT_N];
                }
            }
        }
        if (!p.sched) break;
    }
}


// ---- pair shape: one ciphertext per cluster of two CTAs (br_phases.cuh: "pair shape") -------------------------------
// Lowest latency for batches up to 3/8 of the SM count (capi.cu: pair_max).  No work queue (one cluster per ciphertext,
// one wave or plain hardware queueing of clusters), blind rotation only (`plain` external products take the single-CTA shapes).
// Dynamic shared memory is requested well above what the shape needs so that the two CTAs of a cluster can never
// share an SM.
constexpr size_t BR_PAIR_SMEM_USED = (size_t)PAIR_POLYS * POLY_STRIDE * sizeof(u64) + 2 * NTT_N * sizeof(u64) + NTT_N * sizeof(i32) + 64 +
                                     (size_t)PAIR_KEY_PLANES * NTT_N * sizeof(u64);
constexpr size_t BR_PAIR_SMEM_BYTES = 120 * 1024;
static_assert(BR_PAIR_SMEM_USED <= BR_PAIR_SMEM_BYTES, "pair shape shared memory");

NB_D unsigned cluster_cta_rank()
{
    unsigned r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
// the address of `ptr` (this CTA's shared memory, generic) in CTA `rank` of the cluster
NB_D u64 *cluster_map_shared(u64 *ptr, unsigned rank)
{
    unsigned long long out;
    asm volatile("mapa.u64 %0, %1, %2;" : "=l"(out) : "l"((unsigned long long)ptr), "r"(rank));
    return reinterpret_cast<u64 *>(out);
}
// the same for a 32-bit shared-window address (what st.async and mbarrier operands take)
NB_D unsigned cluster_map_shared_u32(unsigned saddr, unsigned rank)
{
    unsigned out;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(out) : "r"(saddr), "r"(rank));
    return out;
}
// cluster-wide barrier; orders this CTA's remote stores before the peer's loads after it
NB_D void cluster_barrier()
{
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
NB_D void mbar_init(unsigned bar, unsigned count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory"); }
NB_D void mbar_expect_tx(unsigned bar, unsigned bytes)
{
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(bar), "r"(bytes) : "memory");
}
NB_D void mbar_wait(unsigned bar, unsigned parity)
{
    asm volatile("{\n\t.reg .pred p;\n\t"
                 "NB_MBAR_WAIT:\n\t"
                 "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
                 "@!p bra NB_MBAR_WAIT;\n\t}" ::"r"(bar), "r"(parity) : "memory");
}
// 16 bytes into the peer's shared memory, completion counted on the peer's mbarrier
NB_D void st_async_peer(unsigned raddr, u64 x, u64 y, unsigned rbar)
{
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v2.b64 [%0], {%1, %2}, [%3];" ::"r"(raddr), "l"(x), "l"(y), "r"(rbar) : "memory");
}

// ASYNC: the partial sums travel as st.async stores that count their bytes on an mbarrier of the receiving CTA, one
// per step parity, which the receiver arms at the top of the step and waits for after its own MAC: no cluster-wide
// barrier in the step loop.  Flow control is the data dependence itself (br_phases.cuh: pair shape).
// !ASYNC: plain remote stores and one barrier.cluster per step -- ptxas implements its release / acquire with a
// GPU-scope memory barrier and an L1 invalidation, which is why the other variant exists; kept as the reference
// implementation (NUFHE_B200_PAIR_ASYNC=0).
// LUT: the programmable bootstrap, as in blind_rotate_kernel.
template <bool ASYNC, bool LUT = false>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(PAIR_THREADS, 1)
blind_rotate_pair_kernel(BlindRotateArgs p, const u64 *__restrict__ twd_fwd_g, const u64 *__restrict__ twd_inv_g)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ __align__(8) unsigned long long s_bar[2];
    u64 *w = reinterpret_cast<u64 *>(smem_raw);
    u64 *twd_fwd = w + PAIR_POLYS * POLY_STRIDE, *twd_inv = twd_fwd + NTT_N;
    i32 *acc = reinterpret_cast<i32 *>(twd_inv + NTT_N);       // this CTA's accumulator polynomial
    int *rot = reinterpret_cast<int *>(acc + NTT_N);           // [2], 64 bytes reserved
    // this CTA's key planes of the current step: [j * 2 + mo] and, rank 0 only, the two correction planes
    u64 *key = reinterpret_cast<u64 *>(reinterpret_cast<unsigned char *>(rot) + 64);
    const int tid = threadIdx.x;
    const int rank = (int)cluster_cta_rank();
    const size_t c = blockIdx.x >> 1;                          // grid = 2 x batch
    // The key row of step i + 1 is requested (cp.async, 16 bytes per request) by the warps that have no work in the
    // middle inverse pass of step i and lands during the last one: the MAC then reads shared memory instead of waiting
    // for the L2, whose latency a step of 8 warps cannot hide -- and which every CTA of the launch asks for the same
    // lines at the same time.
    const int key_planes = rank == 0 ? PAIR_KEY_PLANES : 4;
    auto stage_key = [&](int step, int t, int nthreads) {
        const u64 *row = p.bk + (size_t)step * BK_ROW_U64;
        for (int x = t; x < key_planes * (NTT_N / 2); x += nthreads) {
            const int pl = x >> 9, e = (x & 511) * 2;
            const int src = pl < 4 ? rank * 4 + pl : 4 + pl;      // planes 8, 9: corrections
            cp_async16(key + pl * NTT_N + e, row + (size_t)src * NTT_N + e);
        }
        cp_async_commit();
    };
    if (p.n > 0) stage_key(0, tid, PAIR_THREADS);
    for (int i = tid; i < NTT_N; i += PAIR_THREADS) {
        twd_fwd[i] = twd_fwd_g[i]; twd_inv[i] = twd_inv_g[i];
        acc[i] = br_initial_acc<LUT>(p, c, rank, i);
    }
    const unsigned bar0 = (unsigned)__cvta_generic_to_shared(s_bar);
    if (tid == 0) {
        rot[0] = br_rotation<LUT>(p, c, 0);
        if (ASYNC) {
            mbar_init(bar0, 1); mbar_init(bar0 + 8, 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
    }
    u64 *w_peer = cluster_map_shared(w, (unsigned)(rank ^ 1));
    const unsigned w_peer32 = cluster_map_shared_u32((unsigned)__cvta_generic_to_shared(w), (unsigned)(rank ^ 1));
    const unsigned bar_peer = cluster_map_shared_u32(bar0, (unsigned)(rank ^ 1));
    cp_async_wait<0>();
    cluster_barrier();                                         // the peer is running, its barriers are initialised

    const u64 *corr2 = rank == 0 ? key + 4 * NTT_N : nullptr;
    for (int i = 0; i < p.n; i++) {
        const int par = i & 1;
        const int *r = rot + par;
        int next = 0;
        if (tid == 0) {
            if (ASYNC) mbar_expect_tx(bar0 + 8 * par, PAIR_EXCHANGE_BYTES);
            if (i + 1 < p.n) next = br_rotation<LUT>(p, c, i + 1);
        }
        pair_fwd1(tid, acc, w, twd_fwd, r);
        __syncthreads();
        pair_fwd2(tid, w);
        __syncthreads();
        {
            u64 v[16];
            pair_fwd3_load(tid, w, v);
            __syncthreads();                                   // in place: all loads before any store
            pair_fwd3_finish(tid, w, v);
        }
        __syncthreads();
        if (ASYNC) {
            const unsigned rb = bar_peer + 8 * par;
            pair_mac<true>(tid, w, [=](int off, u64 x, u64 y) { st_async_peer(w_peer32 + 8u * (unsigned)off, x, y, rb); },
                           key, corr2, rank, par);
            __syncthreads();                                   // this CTA's own partial sums; the key planes are free
        } else {
            pair_mac<true>(tid, w, [=](int off, u64 x, u64 y) { st2(w_peer + off, x, y); }, key, corr2, rank, par);
            cluster_barrier();
        }
        if (ASYNC) mbar_wait(bar0 + 8 * par, (unsigned)(i >> 1) & 1u);       // the peer's partial sums have landed
        pair_inv3_a(tid, w, par);
        __syncthreads();
        pair_inv3_b(tid, w, par);
        __syncthreads();
        if (tid < PAIR_INV_WORKERS) pair_inv2(tid, w, par);
        else if (i + 1 < p.n) stage_key(i + 1, tid - PAIR_INV_WORKERS, PAIR_THREADS - PAIR_INV_WORKERS);
        __syncthreads();
        pair_inv1_a(tid, w, twd_inv, par);
        __syncthreads();
        pair_inv1_b(tid, acc, w, par);
        cp_async_wait<0>();                                    // the staged key row, before the barrier that ends the step
        if (tid == 0) rot[par ^ 1] = next;
        __syncthreads();
    }

    if constexpr (LUT) {
        // samples j = 0 .. 2^L - 1 into rows c * 2^L + j: masks from polynomial 0, bodies from polynomial 1
        const int L = p.log2_outputs;
        for (int e = tid; e < NTT_N << L; e += PAIR_THREADS) {
            const int j = e >> 10, x = e & (NTT_N - 1);
            const size_t row = (c << L) + j;
            if (rank == 0) p.out_a[row * NTT_N + x] = lut_tail_a(acc, j, x);
            else if (x == 0) p.out_b[row] = acc[j];
        }
    } else {
        for (int x = tid; x < NTT_N; x += PAIR_THREADS) {
            if (p.accum_out) p.accum_out[(c * 2 + rank) * NTT_N + x] = acc[x];
            if (p.extract) {
                // sample extraction (tlwe_gpu.mako:63-82; blind_rotate.mako:213-224): a from polynomial 0, b from polynomial 1
                if (rank == 0) p.out_a[c * NTT_N + x] = x == 0 ? acc[0] : (i32)(0u - (u32)acc[NTT_N - x]);
                else if (x == 0) p.out_b[c] = acc[0];
            }
        }
    }
    // nothing is in flight towards this CTA (it has waited for every exchange) and nothing it sent is unreceived
    // while the peer still runs, but the peer's shared memory must outlive the stores addressed to it: both leave together
    cluster_barrier();
}

// ---- the separate kernels of the reference's multi-kernel bootstrap (bootstrap.py:96-196) ---------------
// They exist so that `single_kernel_bootstrap=False` and callers of the inner seams (SURVEY 8b) get the same
// functions with the same results; the fused kernel above does all of this in shared memory.
//
// ShiftTorusPolynomial (polynomials_gpu.mako:18-77; polynomials_cpu.py:25-59): result = X^e * source with
// e = power (mode 2), 2N - power (mode 0, `invert_powers`), or result = (X^power - 1) * source (mode 1,
// `minus_one`).  One power per group of `polys_per_power` consecutive polynomials, read from
// powers[group * powers_stride + power_idx] (the reference's `powers_view`).
__global__ void shift_torus_polynomial_kernel(i32 *__restrict__ result, const i32 *__restrict__ source,
                                              const i32 *__restrict__ powers, size_t powers_stride, size_t power_idx,
                                              int polys_per_power, int mode, int n_log2, size_t polys)
{
    const int N = 1 << n_log2;
    const size_t total = polys << n_log2;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t poly = i >> n_log2;
        const int idx = (int)(i & (N - 1));
        int pw = powers[(poly / polys_per_power) * powers_stride + power_idx];
        if (mode == 0) pw = 2 * N - pw;
        pw &= 2 * N - 1;
        const int ar = pw & (N - 1);
        const bool flip = pw >= N;
        const i32 src = source[poly * N + ((idx - ar) & (N - 1))];
        const bool neg = (idx < ar) != flip;
        u32 v = neg ? 0u - (u32)src : (u32)src;
        if (mode == 1) v -= (u32)source[poly * N + idx];
        result[i] = (i32)v;
    }
}

// TLweNoiselessTrivial (tlwe_gpu.py:32-74; tlwe_cpu.py:26-38): acc = (0, ..., 0, mu), variances 0
__global__ void tlwe_noiseless_trivial_kernel(i32 *__restrict__ acc, float *__restrict__ cv, const i32 *__restrict__ mu,
                                              int mask_size, int n_log2, size_t batch)
{
    const int N = 1 << n_log2;
    const size_t per = (size_t)(mask_size + 1) << n_log2, total = batch * per;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t c = i / per, r = i % per;
        const int poly = (int)(r >> n_log2), x = (int)(r & (N - 1));
        acc[i] = poly == mask_size ? mu[c * N + x] : 0;
        if (cv && i < batch) cv[i] = 0.f;            // one variance per sample: cv is (B,) (tlwe.py:94-112)
    }
}

// TLweExtractLweSamples (tlwe_gpu.mako:54-84; tlwe_cpu.py:41-60): a[i*N] = acc_i[0], a[i*N + x] = -acc_i[N - x],
// b = acc_k[0]
__global__ void tlwe_extract_lwe_samples_kernel(i32 *__restrict__ out_a, i32 *__restrict__ out_b,
                                                const i32 *__restrict__ acc, int mask_size, int n_log2, size_t batch)
{
    const int N = 1 << n_log2;
    const size_t per = (size_t)mask_size << n_log2, total = batch * per;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t c = i / per, r = i % per;
        const int poly = (int)(r >> n_log2), x = (int)(r & (N - 1));
        const i32 *a = acc + ((c * (mask_size + 1) + poly) << n_log2);
        out_a[i] = x == 0 ? a[0] : (i32)(0u - (u32)a[N - x]);
        if (r == 0) out_b[c] = acc[(c * (mask_size + 1) + mask_size) << n_log2];
    }
}

// Torus32ToPhase (numeric_functions_gpu.py:39-77; numeric_functions_cpu.py:23-37): round to a multiple of
// 2^32 / mspace_size and return the multiple, in [0, mspace_size)
__global__ void t32_to_phase_kernel(i32 *__restrict__ out, const i32 *__restrict__ in, size_t n, u32 mspace_size)
{
    const u32 interv = (u32)((1ull << 32) / mspace_size), half = interv / 2;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        out[i] = (i32)(((u32)in[i] + half) / interv);
}

// Gadget decomposition as its own kernel (TGswPolynomialDecompH, tgsw_gpu.py:31-54; tgsw_cpu.py:26-49):
// out[poly][j][x] = (((in[poly][x] + offset) >> (32 - (j + 1) bg_bit)) & (Bg - 1)) - Bg / 2
__global__ void tgsw_decompose_kernel(i32 *__restrict__ out, const i32 *__restrict__ in, size_t polys, int decomp_length,
                                      int bs_log2_base, i32 offset, int n_log2)
{
    const int N = 1 << n_log2;
    const size_t total = (polys * decomp_length) << n_log2;
    const u32 mask = (1u << bs_log2_base) - 1u, half = 1u << (bs_log2_base - 1);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int x = (int)(i & (N - 1));
        const size_t pj = i >> n_log2;
        const int j = (int)(pj % decomp_length);
        const size_t poly = pj / decomp_length;
        const u32 t = (u32)in[(poly << n_log2) + x] + (u32)offset;
        out[i] = (i32)(((t >> (32 - (j + 1) * bs_log2_base)) & mask) - half);
    }
}

// The point-wise multiply-accumulate of the external product as its own kernel, on the reference's key layout
// (tgsw_gpu.py:58-107; tgsw_cpu.py:52-79): out[b][mo][x] = sum_{mi, j} mul_prepared(tr[b][mi][j][x], bk[mi][j][mo][x])
// for any mask size k (mi, mo <= k) and decomposition length.  bk_row: (k+1, l, k+1, N), Montgomery form.
__global__ void tgsw_mac_kernel(u64 *__restrict__ out, const u64 *__restrict__ tr, const u64 *__restrict__ bk_row,
                                size_t batch, int k1, int decomp_length)
{
    const size_t total = batch * k1 * NTT_N;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int x = (int)(i & (NTT_N - 1));
        const int mo = (int)((i >> 10) % k1);
        const size_t b = (i >> 10) / k1;
        u64 acc = 0;
        for (int mi = 0; mi < k1; mi++)
            for (int j = 0; j < decomp_length; j++) {
                const u64 a = ff_canon(tr[((b * k1 + mi) * decomp_length + j) * NTT_N + x]);
                const u64 w = ff_canon(bk_row[(((size_t)mi * decomp_length + j) * k1 + mo) * NTT_N + x]);
                acc = ff_add(acc, ff_canon(ff_mul_prepared(a, w)));
            }
        out[i] = ff_canon(acc);
    }
}

// tlwe_add_to (tlwe.py:173-175): wrap-around int32 addition, float addition of the variances
__global__ void add_to_kernel(i32 *__restrict__ res, const i32 *__restrict__ src, size_t n, float *__restrict__ res_cv,
                              const float *__restrict__ src_cv, size_t n_cv)
{
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        res[i] = (i32)((u32)res[i] + (u32)src[i]);
        if (res_cv && i < n_cv) res_cv[i] += src_cv[i];
    }
}

// ---- LWE key switch (lwe_gpu.mako:59-118; lwe_cpu.py:62-93) --------------------------------------
// res_a[i] = - sum_{j,k} ks_a[j][k][digit(j,k)][i], res_b = b - sum ks_b[j][k][digit].
//
// The reference gathers one 2000-byte key row per (ciphertext, j, k) from global memory: ~12 MB of key
// per ciphertext.  Here a CTA owns a tile of up to KS_TILE ciphertexts and streams the key ONCE per tile:
// a producer warp moves the key, 32 000 contiguous bytes (four values of k, all four rows) at a time,
// into a ring of four shared-memory slots with cp.async.bulk (TMA, completion on an mbarrier); 8 consumer
// warps (thread t owns output coefficients 2t, 2t+1 of every ciphertext of the tile) pick the row with the
// warp-uniform 2-bit digit and subtract: 3 instructions per (ciphertext, j, k, coefficient).
// Row d = 0 of the key is zero padding (lwe_cpu.py:31-33; the reference kernel skips it, its NumPy closure
// subtracts it): it is streamed like the other rows, so d = 0 needs no branch.
// src = src1 (+ src2) (+ (0, c)) lets gate_mux fold `(0,1/8) + u1 + u2` (gates.py:657-664) into the load.
constexpr int KS_TILE = 32;                 // ciphertexts per CTA (run-time tile <= KS_TILE)
constexpr int KS_CONSUMERS = 256;           // threads 0..249: a[2t], a[2t+1] of every ciphertext of the tile
constexpr int KS_THREADS = KS_CONSUMERS + 64;   // + producer warp (TMA issue) + b/variance warp
constexpr int KS_SLOTS = 4;                 // ring of half-j slots (4 values of k each): two j in flight
constexpr int KS_IN = 1024, KS_N = 500;     // fast-path sizes (api_low_level.py:49-50)
// The variance of a result is a float32 sum of 8192 table entries.  Float addition is not associative, so its shape is
// FIXED: 128 block sums over 8 consecutive input coefficients each (64 terms, added in (j, k) order), then the block
// sums added in block order.  A CTA that owns only a slice of j (small batches, KeyswitchArgs::splits) writes its
// block sums to a scratch array and ks_cv_finalize_kernel adds them; a CTA that owns all of j does both itself.
// Either way the same additions happen in the same order: bit-identical variances for every launch shape, run to run.
constexpr int KS_CV_BLOCK_J = 8;
constexpr int KS_CV_BLOCKS = KS_IN / KS_CV_BLOCK_J;
constexpr int KS_ROW_BYTES = KS_N * 4;
constexpr int KS_SLOT_BYTES = 4 * 4 * KS_ROW_BYTES;   // 4 k x 4 rows
constexpr size_t KS_SMEM_BYTES = (size_t)KS_SLOTS * KS_SLOT_BYTES + (size_t)KS_IN * KS_TILE * 2 + 2 * KS_SLOTS * 8 + 128;

struct KeyswitchArgs {
    const i32 *src1_a, *src1_b, *src2_a, *src2_b;   // (B, in), (B,)
    i32 c;
    const i32 *ks_a, *ks_b;                          // (in, t, base, n), (in, t, base)
    const float *ks_cv;
    i32 *res_a, *res_b;                              // (B, n), (B,)
    float *res_cv;                                   // optional
    int in_size, n, t, log2_base;
    int tile;                                        // ciphertexts per CTA (fast path)
    int splits;                                      // > 1: blockIdx.y takes a slice of j and results are
                                                     // accumulated with integer atomics into zeroed outputs
    float *cv_blocks;                                // splits > 1 and res_cv: (B, KS_CV_BLOCKS) partial variances
    size_t batch;
};

NB_D void mbar_init(u64 *bar, u32 count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count)); }
NB_D void mbar_expect_tx(u64 *bar, u32 bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
NB_D void mbar_arrive(u64 *bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory"); }
NB_D void mbar_wait(u64 *bar, u32 parity)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra WAIT_DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "WAIT_DONE:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
NB_D void bulk_g2s(void *dst, const void *src, u32 bytes, u64 *bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// One tile of the grouped key switch (keyswitch_grouped_kernel): ciphertexts ct0 .. ct0 + nct - 1 (nct <= KS_TILE) of
// the batch, all of one tenant, switched with that tenant's key
struct KsTile {
    const i32 *ks_a, *ks_b;
    const float *ks_cv;
    size_t ct0;
    int nct;
};

// Fast path: in = 1024, n = 500, t = 8, base = 4 (the scheme's parameters, api_low_level.py:49-56).
// GROUPED: CTA x takes tiles[x] (its ciphertexts and key) instead of ciphertexts x * p.tile .. with p's key.
template <bool GROUPED>
NB_D void keyswitch_body(const KeyswitchArgs &p, const KsTile *__restrict__ tiles)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    unsigned char *ring = smem_raw;                                               // [slot][k & 3][row][2000 B]
    unsigned short *digits = reinterpret_cast<unsigned short *>(ring + KS_SLOTS * KS_SLOT_BYTES);  // [j][KS_TILE]
    u64 *full = reinterpret_cast<u64 *>(ring + KS_SLOTS * KS_SLOT_BYTES + KS_IN * KS_TILE * 2);
    u64 *empty = full + KS_SLOTS;

    const int tid = threadIdx.x;
    size_t ct0 = (size_t)blockIdx.x * p.tile;
    int nct = (int)min((size_t)p.tile, p.batch - ct0);
    const i32 *ks_a = p.ks_a, *ks_b = p.ks_b;
    const float *ks_cv = p.ks_cv;
    if constexpr (GROUPED) {
        const KsTile &t = tiles[blockIdx.x];
        ct0 = t.ct0; nct = t.nct; ks_a = t.ks_a; ks_b = t.ks_b; ks_cv = t.ks_cv;
    }
    // slice of the input coefficients handled by this CTA (small batches: split-j over blockIdx.y so that
    // one ciphertext does not stream the whole 65 MB key through a single SM); always an even number of j
    const int j_per = ((KS_IN + p.splits - 1) / p.splits + KS_CV_BLOCK_J - 1) & ~(KS_CV_BLOCK_J - 1);
    const int j_begin = blockIdx.y * j_per;
    const int j_end = min(KS_IN, j_begin + j_per);
    const bool split = p.splits > 1;

    if (tid == 0) {
        for (int s = 0; s < KS_SLOTS; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], KS_CONSUMERS / 32); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // packed digits of the tile: the 8 two-bit digits of coefficient j of ciphertext q in 16 bits
    const u32 prec_offset = 1u << (32 - (1 + 2 * 8));
    const int jn = max(j_end - j_begin, 0);
    for (int idx = tid; idx < KS_TILE * jn; idx += KS_THREADS) {
        const int q = idx / jn, j = j_begin + idx % jn;
        u32 v = 0;
        if (q < nct) {
            v = (u32)p.src1_a[(ct0 + q) * KS_IN + j];
            if (p.src2_a) v += (u32)p.src2_a[(ct0 + q) * KS_IN + j];
            v = (v + prec_offset) >> 16;              // k = 0 in the top bits
        }
        digits[j * KS_TILE + q] = (unsigned short)v;  // ciphertexts beyond nct: digits 0 (results not stored)
    }
    __syncthreads();

    if (tid >= KS_CONSUMERS + 32) {
        // ---- b / variance warp: lane q owns ciphertext q of the tile; the 16-byte (j, k) entries of ks_b and
        // ks_cv are warp-uniform loads.  Runs beside the consumers and never touches the ring.
        const int q = tid - (KS_CONSUMERS + 32);
        u32 accb = 0;
        float cv = 0.f;
        int4 kb = __ldg(reinterpret_cast<const int4 *>(ks_b));
        float4 kc = __ldg(reinterpret_cast<const float4 *>(ks_cv));
        kb = __ldg(reinterpret_cast<const int4 *>(ks_b) + min(j_begin * 8, KS_IN * 8 - 1));
        kc = __ldg(reinterpret_cast<const float4 *>(ks_cv) + min(j_begin * 8, KS_IN * 8 - 1));
        float blk = 0.f;
        for (int jk = j_begin * 8; jk < j_end * 8; jk++) {
            const int4 kb_next = __ldg(reinterpret_cast<const int4 *>(ks_b) + min(jk + 1, KS_IN * 8 - 1));
            const float4 kc_next = __ldg(reinterpret_cast<const float4 *>(ks_cv) + min(jk + 1, KS_IN * 8 - 1));
            const u32 bits = digits[(jk >> 3) * KS_TILE + q];
            const u32 d = (bits >> (14 - 2 * (jk & 7))) & 3u;
            accb -= d == 0 ? (u32)kb.x : d == 1 ? (u32)kb.y : d == 2 ? (u32)kb.z : (u32)kb.w;
            blk += d == 0 ? kc.x : d == 1 ? kc.y : d == 2 ? kc.z : kc.w;
            kb = kb_next; kc = kc_next;
            if ((jk & (8 * KS_CV_BLOCK_J - 1)) == 8 * KS_CV_BLOCK_J - 1) {      // end of a block of 8 coefficients
                if (split) { if (p.cv_blocks && q < nct) p.cv_blocks[(ct0 + q) * KS_CV_BLOCKS + (jk >> 6)] = blk; }
                else cv += blk;
                blk = 0.f;
            }
        }
        if (q < nct) {
            u32 b = (u32)p.src1_b[ct0 + q] + (p.src2_b ? (u32)p.src2_b[ct0 + q] : 0u) + (u32)p.c;
            if (!split) {
                p.res_b[ct0 + q] = (i32)(b + accb);
                if (p.res_cv) p.res_cv[ct0 + q] = cv;
            } else {
                atomicAdd(reinterpret_cast<unsigned int *>(p.res_b + ct0 + q), (blockIdx.y == 0 ? b : 0u) + accb);
            }
        }
        return;
    }
    if (tid >= KS_CONSUMERS) {
        // ---- producer warp: one lane streams the key, 32 000 bytes per slot ------------------------
        if (tid == KS_CONSUMERS) {
            for (int j = j_begin; j < j_end; j++) {
                const u32 parity = ((((j - j_begin) >> 1) & 1)) ^ 1;
#pragma unroll 1
                for (int h = 0; h < 2; h++) {
                    const int slot = 2 * (j & 1) + h;
                    mbar_wait(&empty[slot], parity);  // first pass: passes immediately (phase -1 "complete")
                    mbar_expect_tx(&full[slot], KS_SLOT_BYTES);
                    bulk_g2s(ring + slot * KS_SLOT_BYTES, ks_a + (size_t)(j * 8 + 4 * h) * 4 * KS_N, KS_SLOT_BYTES,
                             &full[slot]);
                }
            }
        }
        return;
    }

    // ---- consumers -------------------------------------------------------------------------------
    const bool is_a = tid < KS_N / 2;
    const int lane = tid & 31;
    u32 acc0[KS_TILE], acc1[KS_TILE];
#pragma unroll
    for (int q = 0; q < KS_TILE; q++) { acc0[q] = 0; acc1[q] = 0; }
    // byte offset of this thread's pair inside a key row; idle threads read pair 0 harmlessly
    const u32 col_off = is_a ? (u32)tid * 8u : 0u;
    const u32 ring_base = smem_u32(ring);

    for (int j = j_begin; j < j_end; j++) {
        u32 w[KS_TILE / 2];                            // packed digits of the tile for this j (64 bytes)
        {
            const uint4 *dg = reinterpret_cast<const uint4 *>(digits + j * KS_TILE);
#pragma unroll
            for (int x = 0; x < KS_TILE / 8; x++) {
                uint4 t = dg[x];
                w[4 * x] = t.x; w[4 * x + 1] = t.y; w[4 * x + 2] = t.z; w[4 * x + 3] = t.w;
            }
        }
        const u32 parity = ((j - j_begin) >> 1) & 1;
        const u32 jbase = ring_base + (j & 1) * (2 * KS_SLOT_BYTES) + col_off;
#pragma unroll
        for (int k = 0; k < 8; k++) {
            if ((k & 3) == 0) mbar_wait(&full[2 * (j & 1) + (k >> 2)], parity);
            const u32 base = jbase + k * (4 * KS_ROW_BYTES);
            {
#pragma unroll
                for (int q = 0; q < KS_TILE; q++) {
                    const u32 d = (w[q >> 1] >> (16 * (q & 1) + 14 - 2 * k)) & 3u;
                    const u32 addr = d * (u32)KS_ROW_BYTES + base;
                    u32 v0, v1;
                    asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v0), "=r"(v1) : "r"(addr));
                    acc0[q] -= v0;
                    acc1[q] -= v1;
                }
            }
            if ((k & 3) == 3) {
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[2 * (j & 1) + (k >> 2)]);
            }
        }
    }

#pragma unroll
    for (int q = 0; q < KS_TILE; q++) {
        if (q < nct) {
            if (is_a) {
                if (!split) {
                    p.res_a[(ct0 + q) * KS_N + 2 * tid] = (i32)acc0[q];
                    p.res_a[(ct0 + q) * KS_N + 2 * tid + 1] = (i32)acc1[q];
                } else {
                    atomicAdd(reinterpret_cast<unsigned int *>(p.res_a + (ct0 + q) * KS_N + 2 * tid), acc0[q]);
                    atomicAdd(reinterpret_cast<unsigned int *>(p.res_a + (ct0 + q) * KS_N + 2 * tid + 1), acc1[q]);
                }
            }
        }
    }
}

__global__ void __launch_bounds__(KS_THREADS, 1) keyswitch_kernel(KeyswitchArgs p) { keyswitch_body<false>(p, nullptr); }

// the grouped key switch (nb_mk_keyswitch): one tile table entry per CTA
__global__ void __launch_bounds__(KS_THREADS, 1) keyswitch_grouped_kernel(KeyswitchArgs p, const KsTile *__restrict__ tiles)
{
    keyswitch_body<true>(p, tiles);
}

// second half of the fixed-shape variance sum for split launches: one thread per ciphertext adds its block sums in order
__global__ void ks_cv_finalize_kernel(float *__restrict__ res_cv, const float *__restrict__ cv_blocks, size_t batch)
{
    const size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= batch) return;
    const float4 *src = reinterpret_cast<const float4 *>(cv_blocks + c * KS_CV_BLOCKS);
    float cv = 0.f;
#pragma unroll 8
    for (int m = 0; m < KS_CV_BLOCKS / 4; m++) {
        const float4 v = src[m];
        cv += v.x; cv += v.y; cv += v.z; cv += v.w;
    }
    res_cv[c] = cv;
}

// ---- the key switch as a tensor-core GEMM (DESIGN.md section 4): res = -OneHot . Key mod 2^32.
// OneHot has one row per ciphertext and one column per (j, k, d >= 1): 1 where digit (j, k) equals d (row d = 0 of a
// generated key is zero padding, so it is dropped: nb_ks_prepare registers only keys whose d = 0 rows are zero).
// Key has those 24 576 rows and 512 columns (ks_a, then ks_b in column 500, then zeros), split into its 4 byte planes,
// which become 4 x 512 u8 columns.  Every plane sum is at most 8192 * 255 < 2^21, so the u8 x u8 -> s32 products are
// exact and sum_p S_p << 8p is the key switch's sum mod 2^32.
// Tiles: a CTA takes KM_M = 256 ciphertexts (4 consumer warpgroups of 64) and one N tile of 128 GEMM columns: output
// columns 32 nt .. 32 nt + 31, in all 4 planes (plane p in GEMM columns 32p .. 32p + 31), so one thread holds the 4
// plane sums of each of its outputs.  K runs in KM_GROUPS stages of 96: stage G holds j = G + 256 tig (tig < 4), d
// (one per k32 chunk) and k, in the order that makes thread (g, tig) of a warp build its A fragments from the digits of
// one coefficient j per row: byte e of register half h of chunk c is [digit(j, 4h + 3 - e) == c + 1] (ks_mma_k_index).
constexpr int KM_M = 256;                       // ciphertexts per CTA
constexpr int KM_NT = 128;                      // GEMM columns per CTA: 32 outputs x 4 byte planes
constexpr int KM_NTILES = 512 / 32;             // N tiles over the 512 padded output columns
constexpr int KM_GROUPS = KS_IN / 4;            // K stages: 4 coefficients j (96 rows of K) each
constexpr int KM_STAGE_BYTES = 96 * KM_NT;      // one stage of one N tile: 3 chunks of [16 x 8 rows][2 x 16 B]
constexpr int KM_STAGES = 8;                    // TMA ring depth
constexpr int KM_CONSUMERS = 4 * 128;
constexpr int KM_THREADS = KM_CONSUMERS + 128;  // + producer warpgroup (one lane issues the copies)
// registers per thread after setmaxnreg: the producer warpgroup gives back what the consumers' 64 accumulators need
// (640 threads launch with 96 each)
constexpr int KM_PRODUCER_REGS = 24, KM_CONSUMER_REGS = 112;
constexpr size_t KM_SMEM_BYTES = (size_t)KM_STAGES * KM_STAGE_BYTES + 2 * KM_STAGES * 8;
constexpr size_t KM_PLANES_BYTES = (size_t)KM_NTILES * KM_GROUPS * KM_STAGE_BYTES;   // 50 331 648

// The row of the key (j, k, d) and the byte position in the prepared layout of K index `kpos` (0 .. 95) of stage G:
// chunk c = kpos / 32, half h = (kpos / 16) & 1, tig = (kpos / 4) & 3, e = kpos & 3.
NB_HD void ks_mma_k_index(int G, int kpos, int *j, int *k, int *d)
{
    const int c = kpos >> 5, h = (kpos >> 4) & 1, tig = (kpos >> 2) & 3, e = kpos & 3;
    *j = G + KM_GROUPS * tig;
    *k = 4 * h + 3 - e;
    *d = c + 1;
}
// byte offset in the prepared key of (N tile nt, stage G, GEMM column col < 128, K index kpos < 96): chunks of 32 K
// rows in the no-swizzle K-major layout of wgmma, core matrices of 8 columns x 16 bytes, the two K halves of a group
// of 8 columns side by side (leading byte offset 128), groups of 8 columns 256 bytes apart (stride byte offset)
NB_HD size_t ks_mma_offset(int nt, int G, int col, int kpos)
{
    return ((size_t)nt * KM_GROUPS + G) * KM_STAGE_BYTES + (size_t)(kpos >> 5) * (32 * KM_NT) + (col >> 3) * 256 +
           ((kpos >> 4) & 1) * 128 + (col & 7) * 16 + (kpos & 15);
}

struct KeyswitchMmaArgs {
    const i32 *src1_a, *src1_b, *src2_a, *src2_b;   // (B, 1024), (B,); rows 16-byte aligned
    i32 c;
    const uint8_t *planes;                          // nb_ks_prepare
    i32 *res_a, *res_b;                             // (B, 500), (B,)
    size_t batch;
    int splits;                                     // > 1: blockIdx.z takes KM_GROUPS / splits stages, integer
                                                    // atomics into zeroed outputs
};

// nb_ks_prepare: one thread per 4 consecutive bytes of the layout (same j, d, column; k = 4h + 3 .. 4h), and a check
// that the d = 0 rows are zero (their one-hot columns are not in the GEMM)
__global__ void ks_prepare_kernel(const i32 *__restrict__ ks_a, const i32 *__restrict__ ks_b, uint8_t *__restrict__ planes,
                                  int *__restrict__ pad_nonzero)
{
    const size_t words = KM_PLANES_BYTES / 4, pad_words = (size_t)KS_IN * 8 * (KS_N + 1);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < words + pad_words; i += (size_t)gridDim.x * blockDim.x) {
        if (i >= words) {
            const size_t r = (i - words) / (KS_N + 1), x = (i - words) % (KS_N + 1);   // row (j, k, d = 0)
            if ((x < KS_N ? ks_a[r * 4 * KS_N + x] : ks_b[r * 4]) != 0) atomicOr(pad_nonzero, 1);
            continue;
        }
        size_t rest = i;
        const int kq = (int)(rest & 3); rest >>= 2;      // 4-byte group inside the 16-byte core-matrix row
        const int n_in = (int)(rest & 7); rest >>= 3;
        const int h = (int)(rest & 1); rest >>= 1;
        const int n8 = (int)(rest & 15); rest >>= 4;
        const int c = (int)(rest % 3); rest /= 3;
        const int G = (int)(rest % KM_GROUPS), nt = (int)(rest / KM_GROUPS);
        const int col = n8 * 8 + n_in, plane = col >> 5, oc = 32 * nt + (col & 31);
        u32 v = 0;
#pragma unroll
        for (int e = 0; e < 4; e++) {
            int j, k, d;
            ks_mma_k_index(G, 32 * c + 16 * h + 4 * kq + e, &j, &k, &d);
            const size_t row = ((size_t)j * 8 + k) * 4 + d;
            const u32 w = oc < KS_N ? (u32)ks_a[row * KS_N + oc] : oc == KS_N ? (u32)ks_b[row] : 0u;
            v |= ((w >> (8 * plane)) & 0xFFu) << (8 * e);
        }
        *reinterpret_cast<u32 *>(planes + ks_mma_offset(nt, G, col, 32 * c + 16 * h + 4 * kq)) = v;
    }
}

// 4 one-hot bytes from 4 flags at bits 0, 2, 4, 6 (the shifted copies do not overlap below bit 25)
NB_D u32 km_spread(u32 y) { return (y * 0x41041u) & 0x01010101u; }

NB_D void km_wgmma(u32 *d, const u32 *a, u64 desc)
{
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %69, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k32.s32.u8.u8 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,"
        "%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,"
        "%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64, %65, %66, %67}, %68, p;\n}\n"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]),
          "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]),
          "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]),
          "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]),
          "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]),
          "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]),
          "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]),
          "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "r"(1));
}

// the 16-bit digit word of one input coefficient: digit k in bits 14 - 2k, 15 - 2k
NB_D u32 km_digits(u32 a) { return (a + (1u << (32 - (1 + 2 * 8)))) >> 16; }

__global__ void __launch_bounds__(KM_THREADS, 1) keyswitch_mma_kernel(KeyswitchMmaArgs p)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    unsigned char *ring = smem_raw;
    u64 *full = reinterpret_cast<u64 *>(ring + KM_STAGES * KM_STAGE_BYTES);
    u64 *empty = full + KM_STAGES;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int nt = blockIdx.y;
    const int nstages = KM_GROUPS / p.splits, G0 = blockIdx.z * nstages;
    if (tid == 0) {
        for (int s = 0; s < KM_STAGES; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], KM_CONSUMERS / 32); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp >= KM_CONSUMERS / 32) {
        // ---- producer: one lane streams this N tile's stages G0 .. G0 + nstages - 1, 12 KB each
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(KM_PRODUCER_REGS));
        if (warp == KM_CONSUMERS / 32 && lane == 0) {
            const uint8_t *src = p.planes + ((size_t)nt * KM_GROUPS + G0) * KM_STAGE_BYTES;
            for (int s = 0; s < nstages; s++) {
                const int slot = s % KM_STAGES;
                if (s >= KM_STAGES) mbar_wait(&empty[slot], ((s / KM_STAGES) - 1) & 1);
                mbar_expect_tx(&full[slot], KM_STAGE_BYTES);
                bulk_g2s(ring + slot * KM_STAGE_BYTES, src + (size_t)s * KM_STAGE_BYTES, KM_STAGE_BYTES, &full[slot]);
            }
        }
        return;
    }

    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(KM_CONSUMER_REGS));
    // ---- consumers: warpgroup wg owns ciphertexts 64 wg .. 64 wg + 63 of the tile; thread (g, tig) builds the rows
    // g and g + 8 of its warp's 16, for coefficient j = G + 256 tig of stage G
    const int g = lane >> 2, tig = lane & 3;
    const size_t r0 = (size_t)blockIdx.x * KM_M + (warp >> 2) * 64 + (warp & 3) * 16 + g, r1 = r0 + 8;
    const bool v0 = r0 < p.batch, v1 = r1 < p.batch;
    const i32 *s1 = p.src1_a + r0 * KS_IN + KM_GROUPS * tig;          // row g + 8: 8 * KS_IN further
    const i32 *s2 = p.src2_a ? p.src2_a + r0 * KS_IN + KM_GROUPS * tig : nullptr;
    auto load4 = [&](int G, int4 *x0, int4 *x1) {   // src1 (+ src2) of stages G .. G + 3, zeros for rows past the batch
        *x0 = v0 ? __ldg(reinterpret_cast<const int4 *>(s1 + G)) : make_int4(0, 0, 0, 0);
        *x1 = v1 ? __ldg(reinterpret_cast<const int4 *>(s1 + 8 * KS_IN + G)) : make_int4(0, 0, 0, 0);
        if (s2) {
            const int4 y0 = v0 ? __ldg(reinterpret_cast<const int4 *>(s2 + G)) : make_int4(0, 0, 0, 0);
            const int4 y1 = v1 ? __ldg(reinterpret_cast<const int4 *>(s2 + 8 * KS_IN + G)) : make_int4(0, 0, 0, 0);
            x0->x += y0.x; x0->y += y0.y; x0->z += y0.z; x0->w += y0.w;
            x1->x += y1.x; x1->y += y1.y; x1->z += y1.z; x1->w += y1.w;
        }
    };
    // rows past the batch: digit word 0 (all digits 0, no one-hot column set)
    auto pack = [&](i32 a0, i32 a1) { return (v0 ? km_digits((u32)a0) : 0u) | ((v1 ? km_digits((u32)a1) : 0u) << 16); };

    u32 acc[64];
#pragma unroll
    for (int i = 0; i < 64; i++) acc[i] = 0;
    const u32 ring_base = smem_u32(ring);
    // matrix descriptor of chunk 0 of slot 0: start >> 4, leading byte offset 128 >> 4, stride byte offset 256 >> 4,
    // no swizzle
    const u64 desc0 = (u64)((ring_base & 0x3FFFF) >> 4) | ((u64)(128 >> 4) << 16) | ((u64)(256 >> 4) << 32);

    int4 n0, n1;
    load4(G0, &n0, &n1);
    for (int q = 0; q < nstages; q += 4) {
        const u32 w[4] = {pack(n0.x, n1.x), pack(n0.y, n1.y), pack(n0.z, n1.z), pack(n0.w, n1.w)};
        if (q + 4 < nstages) load4(G0 + q + 4, &n0, &n1);
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int s = q + u, slot = s % KM_STAGES;
            u32 a[3][4];
#pragma unroll
            for (int c = 0; c < 3; c++) {
                const u32 x = w[u] ^ (0x55555555u * (u32)(c + 1));
                const u32 z = ~(x | (x >> 1)) & 0x55555555u;      // bit 14 - 2k (+ 16 for row g + 8): digit k == c + 1
                a[c][0] = km_spread((z >> 8) & 0x55u);            // row g, k = 3 .. 0
                a[c][1] = km_spread((z >> 24) & 0x55u);           // row g + 8, k = 3 .. 0
                a[c][2] = km_spread(z & 0x55u);                   // row g, k = 7 .. 4
                a[c][3] = km_spread((z >> 16) & 0x55u);           // row g + 8, k = 7 .. 4
            }
            mbar_wait(&full[slot], (s / KM_STAGES) & 1);
            asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
            for (int c = 0; c < 3; c++)
                km_wgmma(acc, a[c], desc0 + (u64)((slot * KM_STAGE_BYTES + c * 32 * KM_NT) >> 4));
            asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
            asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[slot]);
        }
    }

    // ---- epilogue: acc[4i + 2r + e] is row g + 8r, GEMM column 8i + 2 tig + e; plane p in i = 4p .. 4p + 3
    const bool split = p.splits > 1;
#pragma unroll
    for (int r = 0; r < 2; r++) {
        const size_t row = r ? r1 : r0;
        if (!(r ? v1 : v0)) continue;
#pragma unroll
        for (int i = 0; i < 4; i++) {
            u32 v[2];
#pragma unroll
            for (int e = 0; e < 2; e++) {
                const int x = 4 * i + 2 * r + e;
                v[e] = 0u - (acc[x] + (acc[x + 16] << 8) + (acc[x + 32] << 16) + (acc[x + 48] << 24));
            }
            const int col = 32 * nt + 8 * i + 2 * tig;
            if (col < KS_N) {               // KS_N is even: both columns are mask coefficients
                i32 *dst = p.res_a + row * KS_N + col;
                if (!split) *reinterpret_cast<int2 *>(dst) = make_int2((i32)v[0], (i32)v[1]);
                else {
                    atomicAdd(reinterpret_cast<unsigned int *>(dst), v[0]);
                    atomicAdd(reinterpret_cast<unsigned int *>(dst + 1), v[1]);
                }
            } else if (col == KS_N) {       // column 500: ks_b
                const u32 b = blockIdx.z ? 0u : (u32)p.src1_b[row] + (p.src2_b ? (u32)p.src2_b[row] : 0u) + (u32)p.c;
                if (!split) p.res_b[row] = (i32)(b + v[0]);
                else atomicAdd(reinterpret_cast<unsigned int *>(p.res_b + row), b + v[0]);
            }
        }
    }
}

// The variances beside keyswitch_mma_kernel, in the fixed shape of keyswitch_kernel (KS_CV_BLOCK_J): thread (q, part)
// adds the 64 terms of blocks 16 part .. 16 part + 15 of ciphertext q in (j, k) order, thread (q, 0) adds the 128
// block sums in block order.
__global__ void __launch_bounds__(256) ks_cv_kernel(const i32 *__restrict__ src1_a, const i32 *__restrict__ src2_a,
                                                    const float *__restrict__ ks_cv, float *__restrict__ res_cv, size_t batch)
{
    __shared__ float blocks[KS_CV_BLOCKS][33];
    const int q = threadIdx.x & 31, part = threadIdx.x >> 5;
    const size_t ct = (size_t)blockIdx.x * 32 + q;
    if (ct < batch) {
        for (int bk = part * (KS_CV_BLOCKS / 8); bk < (part + 1) * (KS_CV_BLOCKS / 8); bk++) {
            float blk = 0.f;
            for (int jj = 0; jj < KS_CV_BLOCK_J; jj++) {
                const int j = bk * KS_CV_BLOCK_J + jj;
                u32 v = (u32)src1_a[ct * KS_IN + j];
                if (src2_a) v += (u32)src2_a[ct * KS_IN + j];
                const u32 bits = km_digits(v);
#pragma unroll
                for (int k = 0; k < 8; k++) blk += __ldg(ks_cv + (j * 8 + k) * 4 + ((bits >> (14 - 2 * k)) & 3u));
            }
            blocks[bk][q] = blk;
        }
    }
    __syncthreads();
    if (part == 0 && ct < batch) {
        float cv = 0.f;
        for (int bk = 0; bk < KS_CV_BLOCKS; bk++) cv += blocks[bk][q];
        res_cv[ct] = cv;
    }
}

// Generic decomposition parameters (API parity with LweKeyswitch(…, decomp_length, log2_base)): the
// straightforward per-ciphertext gather.
__global__ void __launch_bounds__(512) keyswitch_generic_kernel(KeyswitchArgs p)
{
    const size_t ct = blockIdx.x;
    const int base = 1 << p.log2_base;
    const u32 prec_offset = 1u << (32 - (1 + p.log2_base * p.t));
    const int i = threadIdx.x;
    const bool is_a = i < p.n, is_b = i == p.n;
    if (!(is_a || is_b)) return;
    u32 acc = 0;
    float cv = 0.f;
    for (int j = 0; j < p.in_size; j++) {
        u32 v = (u32)p.src1_a[ct * p.in_size + j];
        if (p.src2_a) v += (u32)p.src2_a[ct * p.in_size + j];
        const i32 tmp = (i32)(v + prec_offset);
        for (int k = 0; k < p.t; k++) {
            const int d = (tmp >> (32 - (k + 1) * p.log2_base)) & (base - 1);
            const size_t row = ((size_t)j * p.t + k) * base + d;
            if (is_a) acc -= (u32)__ldg(p.ks_a + row * p.n + i);
            else { acc -= (u32)__ldg(p.ks_b + row); cv += __ldg(p.ks_cv + row); }
        }
    }
    if (is_a) p.res_a[ct * p.n + i] = (i32)acc;
    else {
        u32 b = (u32)p.src1_b[ct] + (p.src2_b ? (u32)p.src2_b[ct] : 0u) + (u32)p.c;
        p.res_b[ct] = (i32)(b + acc);
        if (p.res_cv) p.res_cv[ct] = cv;
    }
}

// ---- LWE linear ops (lwe_gpu.mako:123-202): res = c_b * (0,1) + s1 * x1 + s2 * x2 on dense arrays ---
__global__ void lwe_affine_kernel(i32 *res_a, i32 *res_b, const i32 *x1_a, const i32 *x1_b, const i32 *x2_a,
                                  const i32 *x2_b, i32 c, i32 s1, i32 s2, size_t batch, int n)
{
    const size_t total = batch * (size_t)(n + 1);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        if (i < batch * (size_t)n) {
            u32 v = x1_a ? (u32)s1 * (u32)x1_a[i] : 0u;
            if (x2_a) v += (u32)s2 * (u32)x2_a[i];
            res_a[i] = (i32)v;
        } else {
            size_t b = i - batch * (size_t)n;
            u32 v = (u32)c + (x1_b ? (u32)s1 * (u32)x1_b[b] : 0u);
            if (x2_b) v += (u32)s2 * (u32)x2_b[b];
            res_b[b] = (i32)v;
        }
    }
}

// ---- LWE encryption / phase (lwe_gpu.py:186-284, lwe_gpu.mako:205-262; lwe_cpu.py:96-113) and the key-switch key
// (lwe_gpu.py:63-124, lwe_gpu.mako:18-56; lwe_cpu.py:26-59): wrap-around dot products with the binary key.  One warp
// per row, 16-byte loads when the row length allows; nothing is materialised in 64 bits.

// out[i] = add1[i] (+ add2[i]) + sign * <a[i, :], key>   (Torus32, mod 2^32)
//   encrypt: add1 = messages, add2 = Gaussian noise, sign = +1, a = the uniform mask      (b = mu + e + <a, s>)
//   phase:   add1 = b, sign = -1                                                          (b - <a, s>)
__global__ void lwe_dot_kernel(i32 *__restrict__ out, const i32 *__restrict__ a, const i32 *__restrict__ key,
                               const i32 *__restrict__ add1, const i32 *__restrict__ add2, i32 sign, size_t batch, int n)
{
    const int lane = threadIdx.x & 31;
    const size_t warps = ((size_t)gridDim.x * blockDim.x) >> 5;
    for (size_t row = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < batch; row += warps) {
        const i32 *ar = a + row * (size_t)n;
        u32 acc = 0;
        if ((n & 3) == 0) {
            const int4 *a4 = reinterpret_cast<const int4 *>(ar);
            const int4 *k4 = reinterpret_cast<const int4 *>(key);
            for (int j = lane; j < n / 4; j += 32) {
                const int4 x = __ldg(a4 + j), k = __ldg(k4 + j);
                acc += (u32)x.x * (u32)k.x + (u32)x.y * (u32)k.y + (u32)x.z * (u32)k.z + (u32)x.w * (u32)k.w;
            }
        } else {
            for (int j = lane; j < n; j += 32) acc += (u32)__ldg(ar + j) * (u32)__ldg(key + j);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0) {
            u32 v = (u32)sign * acc;
            if (add1) v += (u32)add1[row];
            if (add2) v += (u32)add2[row];
            out[row] = (i32)v;
        }
    }
}

// key-switch key: row (i, j, h) of ks_a / ks_b / ks_cv; h = 0 is the zero padding, h >= 1 encrypts
// in_key[i] * h * 2^(32 - (j + 1) log2_base) under out_key with mask noises_a[i, j, h - 1] and noise noises_b[i, j, h - 1]
__global__ void make_keyswitch_key_kernel(i32 *__restrict__ ks_a, i32 *__restrict__ ks_b, float *__restrict__ ks_cv,
                                          const i32 *__restrict__ in_key, const i32 *__restrict__ out_key,
                                          const i32 *__restrict__ noises_a, const i32 *__restrict__ noises_b,
                                          size_t in_size, int n, int t, int log2_base, float noise_var)
{
    const int base = 1 << log2_base;
    const size_t rows = in_size * t * base;
    const int lane = threadIdx.x & 31;
    const size_t warps = ((size_t)gridDim.x * blockDim.x) >> 5;
    for (size_t row = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
        const int h = (int)(row % base);
        const size_t ij = row / base;
        const int j = (int)(ij % t);
        const size_t i = ij / t;
        i32 *dst = ks_a + row * (size_t)n;
        if (h == 0) {
            for (int x = lane; x < n; x += 32) dst[x] = 0;
            if (lane == 0) { ks_b[row] = 0; ks_cv[row] = 0.f; }
            continue;
        }
        const size_t nrow = ij * (base - 1) + (h - 1);
        const i32 *src = noises_a + nrow * (size_t)n;
        u32 acc = 0;
        for (int x = lane; x < n; x += 32) {
            const i32 v = __ldg(src + x);
            dst[x] = v;
            acc += (u32)v * (u32)__ldg(out_key + x);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0) {
            const u32 message = (u32)in_key[i] * (u32)h * (1u << (32 - (j + 1) * log2_base));
            ks_b[row] = (i32)(message + (u32)noises_b[nrow] + acc);
            ks_cv[row] = noise_var;
        }
    }
}

// ---- seeded masks (DESIGN.md section 10): out[i] = word (first + i) of the ChaCha20 stream (seed, nonce), i < count.
// Each lane computes one 64-byte block; a warp's 32 blocks go through shared memory so that every store instruction of
// the warp writes 32 consecutive words (the kernel is meant to be bound by these writes).  The row stride of 17 words
// keeps the lane-per-block writes into shared memory free of bank conflicts.
struct ChachaSeed { u32 w[8]; };

constexpr int SEEDED_THREADS = 256;

__global__ void __launch_bounds__(SEEDED_THREADS) seeded_uniform_kernel(i32 *__restrict__ out, ChachaSeed seed,
                                                                        u64 nonce, u64 first, u64 count)
{
    __shared__ u32 stage[SEEDED_THREADS / 32][32 * 17];
    const int lane = threadIdx.x & 31;
    u32 *st = stage[threadIdx.x >> 5];
    const u64 blk0 = first >> 4, head = first & 15;
    const u64 blocks = ((first + (count - 1)) >> 4) - blk0 + 1;        // the caller rules out count = 0 and wrapping
    const u64 warps = ((u64)gridDim.x * blockDim.x) >> 5;
    for (u64 wb = (((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 32; wb < blocks; wb += warps * 32) {
        if (wb + lane < blocks) {
            u32 x[16];
            chacha20_block(seed.w, blk0 + wb + lane, nonce, x);
#pragma unroll
            for (int j = 0; j < 16; j++) st[lane * 17 + j] = x[j];
        }
        __syncwarp();
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const int idx = j * 32 + lane;                              // word of the warp's 512-word window
            const u64 w = wb * 16 + idx;                                // stream word - 16 * blk0
            if (w >= head && w - head < count) out[w - head] = (i32)st[(idx >> 4) * 17 + (idx & 15)];
        }
        __syncwarp();
    }
}

// ---- the byte-plane GEMM of public-key encryption (DESIGN.md section 11) and the tree key switch (section 13); layout
// and index arithmetic in plane_gemm.cuh, the operands in pk_layout.cuh (PkSource, PkGemm) and tree_layout.cuh
// (TreeSource, TreeGemm).  Both kernels take the fields of their source or policy as separate parameters, typed by the
// caller with __restrict__ on the pointers: as one struct parameter they make ptxas spill in the encryption GEMM, and
// without __restrict__ its loads of mus leave the read-only path.
// nb_pk_prepare, nb_tree_prepare: the 4 byte planes of W (K x cols), one thread per (column, 4 consecutive k): it reads
// 4 words of W and writes one 32-bit word to each plane.
template <class Src, class... Fields>
__global__ void plane_prepare_kernel(uint8_t *__restrict__ planes, Fields... fields)
{
    const Src src{fields...};
    const u32 K = src.K(), cols = src.cols(), quads = K >> 2;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < (u64)cols * quads; i += (u64)gridDim.x * blockDim.x) {
        const u32 col = (u32)(i / quads), k = (u32)(i % quads) * 4;
        u32 w[4];
#pragma unroll
        for (int j = 0; j < 4; j++) w[j] = src(k + j, col);
#pragma unroll
        for (int p = 0; p < 4; p++) {
            u32 v = 0;
#pragma unroll
            for (int j = 0; j < 4; j++) v |= ((w[j] >> (8 * p)) & 0xFFu) << (8 * j);
            *(u32 *)(planes + plane_offset(p, col, k, K, cols)) = v;
        }
    }
}

template <bool SIGNED_A> NB_D void mma_m16n8k32(i32 *c, const u32 *a, const u32 *b)
{
    if constexpr (SIGNED_A)
        asm("mma.sync.aligned.m16n8k32.row.col.s32.s8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
            : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
    else
        asm("mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
            : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// nb_pk_encrypt, nb_tree_keyswitch: OUT (rows x cols) = A (rows x K) x W (K x cols, 4 byte planes) for the operand
// policy P.  CTA = GEMM_WARPS warps on the same P::NTILES n8 column tiles (blockIdx.y), each warp GEMM_MTILES m16 tiles
// of rows.  Per k-step of 32 a lane loads 2 words of each plane and column tile, forms the A fragment of each of its
// row tiles in registers (P::a_frag), and issues every plane's and column tile's MMA with that fragment, so the four
// plane sums of one output word sit in one thread.  The planes stay in L2 across CTAs.
// plane_gemm_cta is the work of CTA `cta` (rows from cta * MK_TILE_ROWS); nb_mk_tree_keyswitch runs it on a tile.
template <class P>
__device__ __forceinline__ void plane_gemm_cta(const P &op, const uint8_t *__restrict__ planes, u64 rows, u64 cta)
{
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const u64 row0 = (cta * GEMM_WARPS + (threadIdx.x >> 5)) * (16 * GEMM_MTILES);
    if (row0 >= rows) return;
    const u32 K = op.K(), cols = op.cols(), ksteps = K >> 5, col0 = blockIdx.y * (8 * P::NTILES);
    const uint8_t *bcol = planes + plane_offset(0, col0 + g, 0, K, cols);
    const u64 plane_stride = plane_offset(1, 0, 0, K, cols);
    const typename P::Word *arow[GEMM_MTILES][2];
    bool rok[GEMM_MTILES][2];
#pragma unroll
    for (int mt = 0; mt < GEMM_MTILES; mt++)
#pragma unroll
        for (int hr = 0; hr < 2; hr++) {
            const u64 r = row0 + 16 * mt + acc_row(g, 2 * hr);
            rok[mt][hr] = r < rows;
            arow[mt][hr] = op.row(rok[mt][hr] ? r : 0);
        }
    i32 acc[4][GEMM_MTILES][P::NTILES][4];
#pragma unroll
    for (int p = 0; p < 4; p++)
#pragma unroll
        for (int mt = 0; mt < GEMM_MTILES; mt++)
#pragma unroll
            for (int nt = 0; nt < P::NTILES; nt++)
#pragma unroll
                for (int i = 0; i < 4; i++) acc[p][mt][nt][i] = 0;

#pragma unroll P::UNROLL
    for (u32 ks = 0; ks < ksteps; ks++) {
        u32 bf[P::NTILES][4][2];
#pragma unroll
        for (int nt = 0; nt < P::NTILES; nt++)
#pragma unroll
            for (int p = 0; p < 4; p++)
#pragma unroll
                for (int h = 0; h < 2; h++)
                    bf[nt][p][h] = __ldg((const u32 *)(bcol + (u64)8 * nt * K + p * plane_stride + 32 * ks + frag_k(t, h)));
#pragma unroll
        for (int mt = 0; mt < GEMM_MTILES; mt++) {
            u32 af[4];
            op.a_frag(arow[mt], rok[mt], ks, t, af);
#pragma unroll
            for (int nt = 0; nt < P::NTILES; nt++)
#pragma unroll
                for (int p = 0; p < 4; p++) mma_m16n8k32<P::SIGNED_A>(acc[p][mt][nt], af, bf[nt][p]);
        }
    }

#pragma unroll
    for (int mt = 0; mt < GEMM_MTILES; mt++)
#pragma unroll
        for (int nt = 0; nt < P::NTILES; nt++)
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const u64 row = row0 + 16 * mt + acc_row(g, i);
                const u32 col = col0 + 8 * nt + acc_col(t, i);
                if (row >= rows) continue;
                op.store(row, col, combine(acc[0][mt][nt][i], acc[1][mt][nt][i], acc[2][mt][nt][i], acc[3][mt][nt][i]),
                         acc[0][mt][nt][i]);
            }
}

template <class P, class... Fields>
__global__ void __launch_bounds__(GEMM_WARPS * 32) plane_gemm_kernel(const uint8_t *__restrict__ planes, u64 rows,
                                                                     Fields... fields)
{
    plane_gemm_cta(P{fields...}, planes, rows, blockIdx.x);
}

// nb_mk_tree_keyswitch: the tree key switch of several tenants' rows, CTA x on tile x (mk_layout.cuh), which holds at
// most one CTA's rows of one tenant and that tenant's planes.
__global__ void __launch_bounds__(GEMM_WARPS * 32) tree_gemm_mk_kernel(const TreeTile *__restrict__ tiles,
                                                                       const i32 *__restrict__ a, u32 n, u32 cols,
                                                                       i32 *__restrict__ out)
{
    const TreeTile tile = tiles[blockIdx.x];
    plane_gemm_cta(TreeGemm{a + tile.row0 * n, n, cols, out + tile.row0 * cols}, tile.planes, tile.rows, 0);
}

// ---- result packing (DESIGN.md section 12; slot mapping, digits and rounding in pack_layout.cuh).
// nb_pack_digits: LWE masks a (batch, n) row-major -> digit polynomials (groups, n t, N), row i t + j of group g holding
// digit j of a[g N + p][i] at coefficient p.  A transpose: a CTA stages a 32 x 32 tile (32 inputs x 32 mask words) in
// shared memory, loads it along the mask (128 bytes per warp row) and stores it along the slots (128 bytes per warp
// row of a digit polynomial).  The row stride of 33 words keeps the column reads free of bank conflicts.
constexpr int PACK_TILE = 32;
constexpr int PACK_DIGITS_THREADS = 256;

__global__ void __launch_bounds__(PACK_DIGITS_THREADS) pack_digits_kernel(const i32 *__restrict__ a, u32 n, u64 batch,
                                                                           i32 *__restrict__ out)
{
    __shared__ i32 tile[PACK_TILE][PACK_TILE + 1];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const u32 i0 = blockIdx.x * PACK_TILE;
    const u64 c0 = (u64)blockIdx.y * PACK_TILE;                  // 32 consecutive inputs, all in one group
#pragma unroll
    for (int r = ty; r < PACK_TILE; r += PACK_DIGITS_THREADS / 32) {
        const u64 c = c0 + r;
        const u32 i = i0 + tx;
        tile[r][tx] = (c < batch && i < n) ? __ldcs(a + c * n + i) : 0;     // an empty slot has the digits of 0, i.e. 0
    }
    __syncthreads();
    const u64 g = pack_group(c0);
    const u32 p = pack_slot(c0) + tx;
#pragma unroll 4
    for (int q = ty; q < PACK_TILE * PACK_LEVELS; q += PACK_DIGITS_THREADS / 32) {
        const u32 i = i0 + q / PACK_LEVELS;
        const int j = q % PACK_LEVELS;
        if (i < n) out[((g * n + i) * PACK_LEVELS + j) * PACK_N + p] = pack_digit(tile[tx][q / PACK_LEVELS], j);
    }
}

// nb_ntt_mac: out (G, U, N) = sum_r x (G, R, N) . key (R, U, N) on plain-form field elements.  A CTA owns 64 points of
// one group and up to 2 outputs; a lane 2 adjacent points (128-bit loads), each warp a slice r = warp, warp + 16, ...
// of the sum.  The 128-bit products are summed exactly in five 32-bit limbs (mac128) and folded once per warp slice, as
// ff_dot4 does; the 16 slices are added in shared memory.  The digit spectra x are read once with streaming loads, so
// that the key spectra, which every CTA of a group reads, stay in L2.
constexpr int MAC_WARPS = 16;
constexpr int MAC_POINTS = 64;
constexpr int MAC_OUTS = 2;

// ntt_mac_group is the work of a CTA of group g with the key spectra `key`.
__device__ __forceinline__ void ntt_mac_group(const u64 *__restrict__ x, const u64 *__restrict__ key,
                                              u64 *__restrict__ out, u32 R, u32 U, u64 g)
{
#if defined(__CUDA_ARCH__)          // (mac128 and the limb fold exist on the device only)
    __shared__ u64 part[MAC_WARPS][MAC_OUTS][MAC_POINTS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const u32 pt0 = (blockIdx.x % (PACK_N / MAC_POINTS)) * MAC_POINTS, pt = pt0 + 2 * lane;
    const u32 u0 = blockIdx.y * MAC_OUTS, outs = U - u0 < (u32)MAC_OUTS ? U - u0 : (u32)MAC_OUTS;
    u32 acc[MAC_OUTS][2][5];
#pragma unroll
    for (int o = 0; o < MAC_OUTS; o++)
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
            for (int l = 0; l < 5; l++) acc[o][h][l] = 0;
    const u64 *xg = x + g * R * PACK_N + pt;
    const u64 *kg = key + (u64)u0 * PACK_N + pt;
#pragma unroll 4
    for (u32 r = warp; r < R; r += MAC_WARPS) {
        const ulonglong2 xv = __ldcs((const ulonglong2 *)(xg + (u64)r * PACK_N));
#pragma unroll
        for (int o = 0; o < MAC_OUTS; o++) {
            if (o < (int)outs) {
                const ulonglong2 kv = __ldg((const ulonglong2 *)(kg + ((u64)r * U + o) * PACK_N));
                mac128(xv.x, kv.x, acc[o][0][0], acc[o][0][1], acc[o][0][2], acc[o][0][3], acc[o][0][4]);
                mac128(xv.y, kv.y, acc[o][1][0], acc[o][1][1], acc[o][1][2], acc[o][1][3], acc[o][1][4]);
            }
        }
    }
    // fold: 2^128 = -2^32 (mod p), and the carry limb counts at most one per term
#pragma unroll
    for (int o = 0; o < MAC_OUTS; o++)
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const u32 *c = acc[o][h];
            part[warp][o][2 * lane + h] = ff_sub(ff_reduce_limbs(c[0], c[1], c[2], c[3]), (u64)c[4] << 32);
        }
    __syncthreads();
    if (threadIdx.x < MAC_OUTS * MAC_POINTS) {
        const int o = threadIdx.x / MAC_POINTS, q = threadIdx.x % MAC_POINTS;
        if (o < (int)outs) {
            u64 s = part[0][o][q];
#pragma unroll
            for (int w = 1; w < MAC_WARPS; w++) s = ff_add(s, part[w][o][q]);
            out[(g * U + u0 + o) * PACK_N + pt0 + q] = ff_canon(s);     // (the folds leave [0, p])
        }
    }
#endif
}

__global__ void __launch_bounds__(MAC_WARPS * 32) ntt_mac_kernel(const u64 *__restrict__ x, const u64 *__restrict__ key,
                                                                 u64 *__restrict__ out, u32 R, u32 U)
{
    ntt_mac_group(x, key, out, R, U, blockIdx.x / (PACK_N / MAC_POINTS));
}

// nb_mk_ntt_mac: the same with the key spectra of group g at group_keys[g] (mk_layout.cuh: mk_group_keys).
__global__ void __launch_bounds__(MAC_WARPS * 32) ntt_mac_mk_kernel(const u64 *__restrict__ x,
                                                                    const u64 *const *__restrict__ group_keys,
                                                                    u64 *__restrict__ out, u32 R, u32 U)
{
    const u64 g = blockIdx.x / (PACK_N / MAC_POINTS);
    ntt_mac_group(x, group_keys[g], out, R, U, g);
}

// nb_pack_finish: out (G, k+1, N) uint16 = round_16(-C) for the masks, round_16(b_c - C) at the slots of the body.
__global__ void pack_finish_kernel(const i32 *__restrict__ c, const i32 *__restrict__ b, u32 k, u64 batch,
                                   uint16_t *__restrict__ out, u64 total)
{
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (u64)gridDim.x * blockDim.x) {
        const u64 poly = i / PACK_N, g = poly / (k + 1);
        const u32 u = (u32)(poly % (k + 1));
        const u64 cidx = g * PACK_N + (i % PACK_N);
        u32 v = 0u - (u32)c[i];
        if (u == k && cidx < batch) v += (u32)b[cidx];
        out[i] = pack_round16(v);
    }
}

// ---- tree-based programmable bootstrapping (DESIGN.md section 13; index arithmetic in tree_layout.cuh).
// nb_tree_assemble: one CTA per (test vector, polynomial u).  Z_u = sum_m X^(o_m) G_m,u in shared memory, its
// exclusive prefix sums (4 coefficients per thread, a warp scan, then the warp totals), then every coefficient of
// Q_P Z_u as the difference of two prefix sums.  All sums wrap mod 2^32, which is exact.
constexpr int TREE_ASM_THREADS = 256;
static_assert(TREE_ASM_THREADS * 4 == PACK_N, "tree_assemble_kernel: 4 coefficients per thread");

__global__ void __launch_bounds__(TREE_ASM_THREADS) tree_assemble_kernel(const i32 *__restrict__ v,
                                                                          const i32 *__restrict__ b, int bits, u32 k,
                                                                          i32 *__restrict__ tv)
{
    __shared__ u32 z[PACK_N];
    __shared__ u32 ps[PACK_N + 1];
    __shared__ u32 warp_sum[TREE_ASM_THREADS / 32];
    const u64 t = blockIdx.x / (k + 1);
    const u32 u = blockIdx.x % (k + 1);
    const int M = 1 << bits, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int x = tid; x < PACK_N; x += TREE_ASM_THREADS) {
        u32 s = 0;
        for (int m = 0; m < M; m++) {
            bool neg;
            const int d = tree_shift_index(tree_offset(m, bits), x, &neg);
            const u32 gv = tree_glwe_coef(v + ((t * M + m) * (k + 1) + u) * PACK_N, b[t * M + m], u == k, d);
            s += neg ? 0u - gv : gv;
        }
        z[x] = s;
    }
    __syncthreads();
    u32 loc[4], run = 0;
#pragma unroll
    for (int q = 0; q < 4; q++) { loc[q] = run; run += z[4 * tid + q]; }
    u32 incl = run;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const u32 y = __shfl_up_sync(0xffffffffu, incl, off);
        if (lane >= off) incl += y;
    }
    if (lane == 31) warp_sum[warp] = incl;
    __syncthreads();
    u32 base = incl - run;
    for (int w = 0; w < warp; w++) base += warp_sum[w];
#pragma unroll
    for (int q = 0; q < 4; q++) ps[4 * tid + q] = base + loc[q];
    if (tid == TREE_ASM_THREADS - 1) ps[PACK_N] = base + run;
    __syncthreads();
    i32 *out = tv + (t * (k + 1) + u) * PACK_N;
    for (int x = tid; x < PACK_N; x += TREE_ASM_THREADS) out[x] = (i32)tree_window_coef(ps, PACK_N >> bits, x);
}

}  // namespace nb
