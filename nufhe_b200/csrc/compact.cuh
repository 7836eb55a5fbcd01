// compact.cuh -- compact public-key encryption (DESIGN.md section 16; slot mapping, rounding and extraction in
// compact_layout.cuh).  Encryption multiplies the binary polynomial r of each group by the key's k + 1 polynomials
// through the exact NTT (nb_ntt_forward_i32, nb_ntt_mac, nb_ntt_inverse_i32); these two kernels finish it and start
// the server's expansion, which the cloud key's key switch (nb_keyswitch) completes.
#pragma once
#include "compact_layout.cuh"

namespace nb {

// nb_compact_finish: out (G, k+1, N) uint16 = round_16(c + e1) for the masks, round_16(c + e2 + mu_c) at the occupied
// slots of the body and 0 at its empty slots.
__global__ void compact_finish_kernel(const i32 *__restrict__ c, const i32 *__restrict__ e1, const i32 *__restrict__ e2,
                                      const i32 *__restrict__ mus, u32 k, u64 batch, uint16_t *__restrict__ out, u64 total)
{
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (u64)gridDim.x * blockDim.x) {
        const u64 poly = i / PACK_N, g = poly / (k + 1);
        const u32 u = (u32)(poly % (k + 1)), j = (u32)(i % PACK_N);
        const bool body = u == k;
        const u64 cidx = g * PACK_N + j;
        const bool occupied = cidx < batch;
        const u32 noise = body ? (u32)e2[g * PACK_N + j] : (u32)e1[(g * k + u) * PACK_N + j];
        out[i] = compact_coeff((u32)c[i], noise, body, occupied, body && occupied ? (u32)mus[cidx] : 0u);
    }
}

// nb_compact_extract: one pass of groups (G', k+1, N) uint16 -> the extracted masks (rows, k N) and bodies (rows,)
// int32 of its first `rows` slots.  A CTA owns CX_ROWS slots of one group and one mask polynomial u (blockIdx.z): it
// stages A'_u, restored to 32 bits, in shared memory in reversed order, so that the consecutive words of an output row
// read consecutive words of the stage, and writes each row segment u N .. u N + N - 1 with 16-byte streaming stores.
// The reads of a warp hit each bank 4 times; the rows (4 KB each per mask polynomial) are what the kernel waits on.
constexpr int CX_ROWS = 32;
constexpr int CX_THREADS = 256;

__global__ void __launch_bounds__(CX_THREADS) compact_extract_kernel(const uint16_t *__restrict__ data, u32 k, u64 rows,
                                                                     i32 *__restrict__ out_a, i32 *__restrict__ out_b)
{
    __shared__ u32 rev[PACK_N];                                   // rev[N - 1 - i] = A'_u[i]
    const u64 g = blockIdx.y;
    const u32 u = blockIdx.z, p0 = blockIdx.x * CX_ROWS;
    const u64 c0 = g * PACK_N + p0;
    if (c0 >= rows) return;                                       // (uniform over the CTA)
    const uint16_t *grp = data + g * (k + 1) * PACK_N;
    {
        const uint2 w = reinterpret_cast<const uint2 *>(grp + (u64)u * PACK_N)[threadIdx.x];   // 4 coefficients
        const u32 i = 4 * threadIdx.x;
        rev[PACK_N - 1 - i] = pack_unround16((uint16_t)(w.x & 0xffffu));
        rev[PACK_N - 2 - i] = pack_unround16((uint16_t)(w.x >> 16));
        rev[PACK_N - 3 - i] = pack_unround16((uint16_t)(w.y & 0xffffu));
        rev[PACK_N - 4 - i] = pack_unround16((uint16_t)(w.y >> 16));
    }
    __syncthreads();
    const u32 nrows = rows - c0 < (u64)CX_ROWS ? (u32)(rows - c0) : (u32)CX_ROWS;
    const u64 row_words = (u64)k * PACK_N;
    for (u32 q = threadIdx.x; q < nrows * (PACK_N / 4); q += CX_THREADS) {
        const u32 r = q / (PACK_N / 4), j0 = 4 * (q % (PACK_N / 4)), p = p0 + r;
        i32 v[4];
#pragma unroll
        for (int s = 0; s < 4; s++) {
            const u32 x = rev[PACK_N - 1 - compact_extract_src(p, j0 + s)];
            v[s] = (i32)(compact_extract_negated(p, j0 + s) ? 0u - x : x);
        }
        __stcs(reinterpret_cast<int4 *>(out_a + (c0 + r) * row_words + (u64)u * PACK_N + j0), make_int4(v[0], v[1], v[2], v[3]));
    }
    if (u == 0 && threadIdx.x < nrows) out_b[c0 + threadIdx.x] = (i32)pack_unround16(grp[(u64)k * PACK_N + p0 + threadIdx.x]);
}

}  // namespace nb
