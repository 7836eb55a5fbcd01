// pack_layout.cuh -- the index and rounding functions of result packing (DESIGN.md section 12), kept apart from the
// kernels so that g++ compiles them into the host emulator (host_emul.cpp) and the CPU suite checks them:
//   * the slot mapping: input c (C order) goes to group c / N, slot c % N;
//   * the digits of a mask word: t = 2 levels of base 2^8, gadget g_0 = 2^24, g_1 = 2^16, every digit in [-128, 127],
//     d_0 g_0 + d_1 g_1 = round_16(a) mod 2^32;
//   * the 16-bit mod switch of the output coefficients and its inverse.
#pragma once
#include "ff.cuh"

namespace nb {

constexpr int PACK_N = 1024;          // slots per group: the GLWE polynomial degree N
constexpr int PACK_LEVELS = 2;        // t, the decomposition length of the packing key

NB_HD u64 pack_group(u64 c) { return c / PACK_N; }
NB_HD u32 pack_slot(u64 c) { return (u32)(c % PACK_N); }

// w = a + 2^15 + 2^23 + 2^31 (mod 2^32): the rounding offset 2^15 and the offsets 2^7 * g_j that centre each digit
NB_HD u32 pack_digit_word(i32 a) { return (u32)a + 0x80808000u; }
NB_HD i32 pack_digit(i32 a, int j)
{
    const u32 w = pack_digit_word(a);
    return j == 0 ? (i32)(w >> 24) - 128 : (i32)((w >> 16) & 255u) - 128;
}

// x -> round(x / 2^16) mod 2^16, and back
NB_HD uint16_t pack_round16(u32 x) { return (uint16_t)((x + 0x8000u) >> 16); }
NB_HD u32 pack_unround16(uint16_t v) { return (u32)v << 16; }

}  // namespace nb
