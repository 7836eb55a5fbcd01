// pk_layout.cuh -- the operands of public-key encryption (DESIGN.md section 11) for the byte-plane GEMM of
// plane_gemm.cuh, kept apart from the MMA so that g++ compiles them into the host emulator (host_emul.cpp) and the CPU
// suite checks them:
//   * the words of W that nb_pk_prepare splits into planes,
//   * which bits of R each lane feeds to the m16n8k32 u8 A fragments,
//   * where each output word goes.
// Encryption of B messages is (a, b, popcount) = R W with W = [A | b_pk | 1] (m x (n+2)) and R binary (B x m): a GEMM
// with K = m, 0/1 A bytes and npad columns.
#pragma once
#include "plane_gemm.cuh"

namespace nb {

// Columns of W padded to whole n8 tiles: a, then b, then the ones column that counts the bits of R.
NB_HD u32 pk_cols_padded(u32 n) { return (n + 2 + 7) & ~7u; }

// W[k][col] as the 32-bit word the planes split: a[k][col], b[k] in column n, 1 in column n + 1, 0 in the padding.
NB_HD u32 pk_source_word(const i32 *a, const i32 *b, u32 n, u32 k, u32 col)
{
    if (col < n) return (u32)a[(u64)k * n + col];
    if (col == n) return (u32)b[k];
    return col == n + 1 ? 1u : 0u;
}

// A fragment register: the bits k = frag_k(t, h) .. + 3 of the 32-bit R word of its row, as four 0/1 bytes (byte j
// = bit k + j, the lowest byte first).  The shifted copies of the nibble do not overlap, so the product has no carries.
NB_HD u32 pk_a_frag(u32 r_word, int t, int h)
{
    const u32 nib = (r_word >> frag_k(t, h)) & 0xFu;
    return (nib * 0x00204081u) & 0x01010101u;
}

// The source of nb_pk_prepare's planes.
struct PkSource {
    const i32 *a, *b;
    u32 m, n;
    NB_HD u32 K() const { return m; }
    NB_HD u32 cols() const { return pk_cols_padded(n); }
    NB_HD u32 operator()(u32 k, u32 col) const { return pk_source_word(a, b, n, k, col); }
};

// The operand policy of nb_pk_encrypt: A rows are the packed bits of R (m / 32 words per row).
struct PkGemm {
    static constexpr int NTILES = 1;          // n8 column tiles per CTA
    static constexpr bool SIGNED_A = false;   // 0/1 bytes: mma .u8.u8
    static constexpr int UNROLL = 2;          // unroll of the k-step loop
    typedef u32 Word;
    const u32 *r_bits;
    u32 m, n;
    const i32 *mus;
    float row_variance;
    i32 *out_a, *out_b;
    float *out_cv;

    NB_HD u32 K() const { return m; }
    NB_HD u32 cols() const { return pk_cols_padded(n); }
    NB_HD const u32 *row(u64 r) const { return r_bits + r * (m >> 5); }
    // The A registers of k-step ks for rows g (row[0]) and g + 8 (row[1]) of a tile; a row past the batch is zero.
    NB_HD void a_frag(const u32 *const row[2], const bool ok[2], u32 ks, int t, u32 af[4]) const
    {
        const u32 w0 = ok[0] ? ldg(row[0] + ks) : 0u;
        const u32 w1 = ok[1] ? ldg(row[1] + ks) : 0u;
        af[0] = pk_a_frag(w0, t, 0);
        af[1] = pk_a_frag(w1, t, 0);
        af[2] = pk_a_frag(w0, t, 1);
        af[3] = pk_a_frag(w1, t, 1);
    }
    // Columns < n are the mask, column n the body plus mu, column n + 1 the popcount of R's row (its plane-0 sum).
    NB_HD void store(u64 row, u32 col, u32 v, i32 s0) const
    {
        if (col < n) out_a[row * n + col] = (i32)v;
        else if (col == n) out_b[row] = (i32)(v + (u32)mus[row]);
        else if (col == n + 1) out_cv[row] = (float)s0 * row_variance;
    }
};

}  // namespace nb
