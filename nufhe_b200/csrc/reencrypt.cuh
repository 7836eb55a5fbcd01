// reencrypt.cuh -- re-encryption from one client's LWE key to the GLWE key of another's bootstrap key (DESIGN.md section
// 22; index functions in reencrypt_layout.cuh).  nb_reencrypt turns LWE samples (a, b) under s_A into LWE samples under
// the extracted key of S_B with one exact negacyclic product per sample: the key C = (A_C, B_C) encrypts s_A[i] g_j at
// slot 2 i + j, so (0, b) - sum_p d_p extract_p(C) has the phase b - sum_i s_A[i] round_16(a_i).  The cloud key's key
// switch (nb_keyswitch) then takes the samples to s_B.
//
// A CTA takes tiles of up to NTT_SWEEP_POLYS consecutive rows of one key and runs the stand-alone transforms' three
// passes (br_phases.cuh) on them, 64 threads per row:
//   1. every thread forms 16 coefficients of -D from the row's mask (the digits of a_i, read from global memory) and
//      adds its terms of the body dot product;
//   2. the forward passes, then the product with the key's mask spectrum in the pass layout (ntt_pair_position);
//   3. the inverse passes, the product staged in shared memory as int32, and the output mask written as 16-byte words.
// Every coefficient of D . A_C is below n t 128 2^31 < p / 2 in magnitude, so the field product is exact mod 2^32.
#pragma once
#include "kernels.cuh"
#include "reencrypt_layout.cuh"

namespace nb {

struct ReencTile {
    const u64 *spectrum;        // NTT of the key's mask A_C: N field elements
    const i32 *body;            // the key's body B_C: N words
    u64 row0;                   // first row of the batch
    u32 rows;                   // 1 .. NTT_SWEEP_POLYS
};

// The tiles of `counts` (keys entries), written to `out` unless it is null; returns their number.
inline u64 reenc_tiles(const size_t *counts, size_t keys, const u64 *const *spectra, const i32 *const *bodies, ReencTile *out)
{
    u64 n = 0, row = 0;
    for (size_t t = 0; t < keys; row += counts[t], t++)
        for (u64 q = 0; q < counts[t]; q += NTT_SWEEP_POLYS, n++)
            if (out) {
                const u64 left = counts[t] - q;
                out[n] = {spectra[t], bodies[t], row + q, (u32)(left < NTT_SWEEP_POLYS ? left : NTT_SWEEP_POLYS)};
            }
    return n;
}

constexpr int REENC_CTAS = 2;        // resident CTAs per SM
NB_HDC size_t reenc_smem_bytes()
{
    return (size_t)NTT_SWEEP_POLYS * POLY_STRIDE * sizeof(u64) + 2 * NTT_N * sizeof(u64) + 2 * NTT_SWEEP_POLYS * sizeof(u32);
}
static_assert(NTT_SWEEP_POLYS * NTT_N * sizeof(i32) <= NTT_SWEEP_POLYS * POLY_STRIDE * sizeof(u64),
              "reencrypt_kernel: the staged products fit the work polynomials");

__global__ void __launch_bounds__(NTT_SWEEP_THREADS, REENC_CTAS)
reencrypt_kernel(const ReencTile *__restrict__ tiles, u64 ntiles, const i32 *__restrict__ a, const i32 *__restrict__ b,
                 u32 n, i32 *__restrict__ out_a, i32 *__restrict__ out_b, const u64 *__restrict__ twd_fwd_g,
                 const u64 *__restrict__ twd_inv_g)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    u64 *w = reinterpret_cast<u64 *>(smem_raw);
    u64 *twd_fwd = w + NTT_SWEEP_POLYS * POLY_STRIDE;
    u64 *twd_inv = twd_fwd + NTT_N;
    u32 *body_part = reinterpret_cast<u32 *>(twd_inv + NTT_N);       // [row][warp of the row]
    i32 *staged = reinterpret_cast<i32 *>(w);                        // the products, once the inverse has read w
    const int tid = threadIdx.x, pl = tid >> 6, j2 = tid & 63;
    for (int i = tid; i < NTT_N; i += NTT_SWEEP_THREADS) {
        twd_fwd[i] = twd_fwd_g[i];
        twd_inv[i] = twd_inv_g[i];
    }
    const int pos = ntt_pair_position(tid);
    for (u64 ti = blockIdx.x; ti < ntiles; ti += gridDim.x) {
        const ReencTile tile = tiles[ti];
        const bool live = (u32)pl < tile.rows;
        const u64 row = tile.row0 + (live ? pl : 0);
        {   // -D in the pass-1 order x[j1] = coefficient 64 j1 + j2, and this thread's terms of sum_p d_p B_C[p]
            const i32 *ar = a + row * n;
            i32 x[16];
            u32 part = 0;
#pragma unroll
            for (int j1 = 0; j1 < 16; j1++) {
                const u32 c = 64 * j1 + j2;
                x[j1] = live ? reenc_digit_coeff(ar, n, c) : 0;
                const i32 d = reenc_negated(reenc_coeff(c)) ? -x[j1] : x[j1];
                part += (u32)d * (u32)__ldg(tile.body + reenc_coeff(c));
            }
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) part += __shfl_xor_sync(0xffffffffu, part, off);
            __syncthreads();            // the previous tile's stores have read `staged` (which aliases w) and body_part
            if ((tid & 31) == 0) body_part[2 * pl + ((tid >> 5) & 1)] = part;
            phase_fwd1_i32(tid, x, w, twd_fwd);
        }
        __syncthreads();
        { const int g = tid >> 6, x = tid & 63; phase_fwd2(x >> 4, x & 15, g, w); }
        __syncthreads();
        { const int u = tid & 3, r = (tid >> 2) & 15, p = tid >> 6; phase_fwd3(p, r, u, w); }
        __syncthreads();
        {   // pointwise product with the key's mask spectrum: this thread's natural points 2t, 2t+1, 2t+512, 2t+513
            const ulonglong2 s_lo = __ldg(reinterpret_cast<const ulonglong2 *>(tile.spectrum) + tid);
            const ulonglong2 s_hi = __ldg(reinterpret_cast<const ulonglong2 *>(tile.spectrum) + tid + 256);
#pragma unroll
            for (int q = 0; q < NTT_SWEEP_POLYS; q++) {
                u64 a0, a1, b0, b1;
                ld2(w + q * POLY_STRIDE + pos, a0, a1);                       // k = 2t, 2t + 512
                ld2(w + q * POLY_STRIDE + pos + 8 * ROW_STRIDE, b0, b1);      // k = 2t + 1, 2t + 513
                st2(w + q * POLY_STRIDE + pos, ff_canon(ff_mul(a0, s_lo.x)), ff_canon(ff_mul(a1, s_hi.x)));
                st2(w + q * POLY_STRIDE + pos + 8 * ROW_STRIDE, ff_canon(ff_mul(b0, s_lo.y)), ff_canon(ff_mul(b1, s_hi.y)));
            }
        }
        __syncthreads();
        { const int u = tid & 3, r = (tid >> 2) & 15, p = tid >> 6; phase_inv3(p, r, u, w); }
        __syncthreads();
        { const int g = tid >> 6, x = tid & 63; phase_inv2(x >> 4, x & 15, g, w); }
        __syncthreads();
        i32 y[16];
        phase_inv1_i32(tid, y, w, twd_inv);
        __syncthreads();
#pragma unroll
        for (int j1 = 0; j1 < 16; j1++) staged[pl * NTT_N + 64 * j1 + j2] = y[j1];
        __syncthreads();
        // output: mask words 4 t .. 4 t + 3 of every live row (one 16-byte store each), and the body
#pragma unroll
        for (int q = 0; q < NTT_SWEEP_POLYS; q++) {
            if ((u32)q < tile.rows) {
                const u32 *prod = reinterpret_cast<const u32 *>(staged + q * NTT_N);
                int4 v;
                v.x = reenc_mask_word(prod, 4 * tid);
                v.y = reenc_mask_word(prod, 4 * tid + 1);
                v.z = reenc_mask_word(prod, 4 * tid + 2);
                v.w = reenc_mask_word(prod, 4 * tid + 3);
                reinterpret_cast<int4 *>(out_a + (tile.row0 + q) * NTT_N)[tid] = v;
            }
        }
        if (tid < (int)tile.rows)
            out_b[tile.row0 + tid] = (i32)((u32)b[tile.row0 + tid] - body_part[2 * tid] - body_part[2 * tid + 1]);
    }
}

}  // namespace nb
