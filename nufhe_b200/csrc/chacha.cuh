// chacha.cuh -- the ChaCha20 block function (RFC 8439 section 2.3, 20 rounds) in the original 64-bit-counter state
// layout, which expands the uniform masks of compressed keys and ciphertexts from a 256-bit seed (DESIGN.md section 10):
//   words 0-3 the constants, 4-11 the seed (8 little-endian words), 12-13 the 64-bit block counter (low word first),
//   14-15 a 64-bit nonce (low word first).
// Word i of the stream (seed, nonce) is word i % 16 of block i / 16.  Compiled by nvcc for seeded_uniform_kernel
// (kernels.cuh) and by g++ into the host emulator (host_emul.cpp), so the CPU suite checks the kernel's arithmetic.
#pragma once
#include "ff.cuh"

namespace nb {

NB_HD u32 chacha_rotl(u32 x, int s)
{
#if defined(__CUDA_ARCH__)
    return __funnelshift_l(x, x, s);
#else
    return (x << s) | (x >> (32 - s));
#endif
}

NB_HD void chacha_quarter_round(u32 &a, u32 &b, u32 &c, u32 &d)
{
    a += b; d ^= a; d = chacha_rotl(d, 16);
    c += d; b ^= c; b = chacha_rotl(b, 12);
    a += b; d ^= a; d = chacha_rotl(d, 8);
    c += d; b ^= c; b = chacha_rotl(b, 7);
}

// out[0..16) = block `counter` of the stream (seed[8], nonce)
NB_HD void chacha20_block(const u32 *seed, u64 counter, u64 nonce, u32 *out)
{
    u32 x[16] = {0x61707865u, 0x3320646eu, 0x79622d32u, 0x6b206574u,
                 seed[0], seed[1], seed[2], seed[3], seed[4], seed[5], seed[6], seed[7],
                 (u32)counter, (u32)(counter >> 32), (u32)nonce, (u32)(nonce >> 32)};
    u32 s[16];
#pragma unroll
    for (int i = 0; i < 16; i++) s[i] = x[i];
#pragma unroll
    for (int r = 0; r < 10; r++) {      // a column round and a diagonal round
        chacha_quarter_round(x[0], x[4], x[8], x[12]);
        chacha_quarter_round(x[1], x[5], x[9], x[13]);
        chacha_quarter_round(x[2], x[6], x[10], x[14]);
        chacha_quarter_round(x[3], x[7], x[11], x[15]);
        chacha_quarter_round(x[0], x[5], x[10], x[15]);
        chacha_quarter_round(x[1], x[6], x[11], x[12]);
        chacha_quarter_round(x[2], x[7], x[8], x[13]);
        chacha_quarter_round(x[3], x[4], x[9], x[14]);
    }
#pragma unroll
    for (int i = 0; i < 16; i++) out[i] = x[i] + s[i];
}

}  // namespace nb
