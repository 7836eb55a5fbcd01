// reencrypt_layout.cuh -- the index functions of re-encryption (DESIGN.md section 22), kept apart from the kernel so that
// g++ compiles them into the host emulator (host_emul.cpp) and the CPU suite checks them:
//   * the key's slots: slot p = 2 i + j of the key sample C encrypts s_A[i] g_j (packing's gadget, pack_layout.cuh);
//   * the digit polynomial: d_p = pack_digit(a_i, j) for p = 2 i + j, and the kernel multiplies C's mask by
//     -D(X) = -d_0 + sum_{p >= 1} d_p X^(N - p), whose coefficient 0 is slot 0 of sum_p d_p X^(-p) C, negated;
//   * the output mask: slot-0 extraction (compact_layout.cuh with p = 0) of P = -D . A_C, which is the mask of
//     (0, b) - sum_p d_p extract_p(C); the body is b - sum_p d_p B_C[p].  All sums wrap mod 2^32.
#pragma once
#include "compact_layout.cuh"

namespace nb {

constexpr int REENC_LEVELS = PACK_LEVELS;      // t = 2: gadget values g_0 = 2^24, g_1 = 2^16

NB_HD u32 reenc_slot(u32 i, int j) { return 2 * i + (u32)j; }

// the coefficient of -D that holds d_p (p = 0 ... N - 1), and whether it holds -d_p; the map is its own inverse
NB_HD u32 reenc_coeff(u32 p) { return (PACK_N - p) & (u32)(PACK_N - 1); }
NB_HD bool reenc_negated(u32 p) { return p == 0; }

// coefficient c of -D for the mask a (n words): 0 beyond the n t digits
NB_HD i32 reenc_digit_coeff(const i32 *a, u32 n, u32 c)
{
    const u32 p = reenc_coeff(c);
    if (p >= REENC_LEVELS * n) return 0;
    const i32 d = pack_digit(a[p / REENC_LEVELS], (int)(p % REENC_LEVELS));
    return reenc_negated(p) ? -d : d;
}

// output mask word j from the product P = -D . A_C (N words)
NB_HD i32 reenc_mask_word(const u32 *prod, u32 j) { return compact_extract(prod, 0, j); }

}  // namespace nb
