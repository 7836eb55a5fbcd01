// pk_layout.cuh -- the index arithmetic of public-key encryption (DESIGN.md section 11), kept apart from the MMA so
// that g++ compiles it into the host emulator (host_emul.cpp) and the CPU suite checks it:
//   * the plane layout nb_pk_prepare writes,
//   * which bits of R and which plane bytes each lane feeds to the m16n8k32 u8 fragments,
//   * the row and column of each accumulator in the epilogue.
// Encryption of B messages is (a, b, popcount) = R W with W = [A | b_pk | 1] (m x (n+2)) and R binary (B x m).  W is
// split into 4 byte planes W = sum_p 2^(8p) W_p; each plane product is an exact u8 x u8 -> s32 GEMM (every sum is at
// most m * 255 < 2^31), and an output word is S0 + 2^8 S1 + 2^16 S2 + 2^24 S3 mod 2^32.
#pragma once
#include "ff.cuh"

namespace nb {

constexpr int PK_WARPS = 4;     // warps per CTA: each its own 64-row slice of the batch, all on the same 8 columns
constexpr int PK_MTILES = 4;    // m16 tiles per warp (64 rows)

// Columns of W padded to whole n8 tiles: a, then b, then the ones column that counts the bits of R.
NB_HD u32 pk_cols_padded(u32 n) { return (n + 2 + 7) & ~7u; }

// Plane p is column-major K x N (the `.col` B operand): byte (k, col) at ((p * npad + col) * m + k).
NB_HD u64 pk_plane_offset(u32 p, u32 col, u32 k, u32 m, u32 npad) { return ((u64)p * npad + col) * m + k; }

// W[k][col] as the 32-bit word the planes split: a[k][col], b[k] in column n, 1 in column n + 1, 0 in the padding.
NB_HD u32 pk_source_word(const i32 *a, const i32 *b, u32 n, u32 k, u32 col)
{
    if (col < n) return (u32)a[(u64)k * n + col];
    if (col == n) return (u32)b[k];
    return col == n + 1 ? 1u : 0u;
}

// The four K values a lane with threadID_in_group t feeds to fragment half h of a k-step: h = 0 is registers a0/a1
// and b0, h = 1 is a2/a3 and b1 (the PTX ISA's logical k offset of 16).  The kernel is free to choose which actual K
// values sit in which logical slot, as long as A and B agree: this order lets each lane read 8 consecutive plane
// bytes per column and 8 consecutive bits of R per row.
NB_HD u32 pk_frag_k(int t, int h) { return 8 * t + 4 * h; }

// A fragment register: the bits k = pk_frag_k(t, h) .. + 3 of the 32-bit R word of its row, as four 0/1 bytes (byte j
// = bit k + j, the lowest byte first).  The shifted copies of the nibble do not overlap, so the product has no carries.
NB_HD u32 pk_a_frag(u32 r_word, int t, int h)
{
    const u32 nib = (r_word >> pk_frag_k(t, h)) & 0xFu;
    return (nib * 0x00204081u) & 0x01010101u;
}

// Accumulator register i (0..3) of lane (groupID g, threadID_in_group t): row g (+8 for i >= 2), column 2t + (i & 1).
NB_HD u32 pk_acc_row(int g, int i) { return g + 8 * (i >> 1); }
NB_HD u32 pk_acc_col(int t, int i) { return 2 * t + (i & 1); }

// The output word of the four plane sums of one (row, column).
NB_HD u32 pk_combine(i32 s0, i32 s1, i32 s2, i32 s3)
{
    return (u32)s0 + ((u32)s1 << 8) + ((u32)s2 << 16) + ((u32)s3 << 24);
}

}  // namespace nb
