// tree_layout.cuh -- the index and sign arithmetic of tree-based programmable bootstrapping (DESIGN.md section 13),
// kept apart from the kernels so that g++ compiles it into the host emulator (host_emul.cpp) and the CPU suite checks
// it:
//   * the LWE -> GLWE key switch V (R, k+1, N) = D (R, n t) x T (n t, (k+1) N) mod 2^32 as the byte-plane GEMM of
//     plane_gemm.cuh: the key words nb_tree_prepare splits into planes, and the signed 8-bit digit fragments a lane
//     forms from two mask words;
//   * the test-vector assembly tv_u = sum_m X^(o_m) Q_P G_m,u (negacyclic) with Q_P = 1 + X + ... + X^(box - 1):
//     Z_u = sum_m X^(o_m) G_m,u first, then the box sum of Z_u from its prefix sums.
#pragma once
#include "pack_layout.cuh"
#include "plane_gemm.cuh"

namespace nb {

// digit rows n t padded to whole k-steps of 32 (the padding rows of the key planes are zero)
NB_HD u32 tree_k_padded(u32 n) { return (n * PACK_LEVELS + 31u) & ~31u; }

// T[kk][col], kk = i t + j, col = u N + x: mask u < k of key row kk (masks (n, t, k, N)) or its body (bodies (n, t, N))
NB_HD u32 tree_key_word(const i32 *masks, const i32 *body, u32 n, u32 k, u32 kk, u32 col)
{
    if (kk >= n * PACK_LEVELS) return 0u;
    const u32 u = col / PACK_N, x = col % PACK_N;
    return u < k ? (u32)masks[((u64)kk * k + u) * PACK_N + x] : (u32)body[(u64)kk * PACK_N + x];
}

// The A fragment register of K values kb .. kb + 3 (kb = 32 ks + frag_k(t, h), even): the digits d_0, d_1 of mask
// words kb / 2 and kb / 2 + 1 as four signed bytes, lowest first.  Byte 3 - j of pack_digit_word is d_j + 128, so the
// signed byte is that byte with its top bit flipped.
NB_HD u32 tree_a_frag(i32 a0, i32 a1)
{
    const u32 w0 = pack_digit_word(a0), w1 = pack_digit_word(a1);
    const u32 v = (w0 >> 24) | (((w0 >> 16) & 0xFFu) << 8) | ((w1 >> 24) << 16) | (((w1 >> 16) & 0xFFu) << 24);
    return v ^ 0x80808080u;
}

// The source of nb_tree_prepare's planes: K = tree_k_padded(n) rows, (k + 1) N columns.
struct TreeSource {
    const i32 *masks, *body;
    u32 n, k;
    NB_HD u32 K() const { return tree_k_padded(n); }
    NB_HD u32 cols() const { return (k + 1) * PACK_N; }
    NB_HD u32 operator()(u32 kk, u32 col) const { return tree_key_word(masks, body, n, k, kk, col); }
};

// The operand policy of nb_tree_keyswitch: A rows are LWE masks of n words, each giving t = 2 signed digits.  Every
// plane sum is at most K * 128 * 255.
struct TreeGemm {
    static constexpr int NTILES = 2;          // n8 column tiles per CTA
    static constexpr bool SIGNED_A = true;    // signed digits: mma .s8.u8
    static constexpr int UNROLL = 1;          // unroll of the k-step loop
    typedef i32 Word;
    const i32 *a;
    u32 n, ncols;
    i32 *out;

    NB_HD u32 K() const { return tree_k_padded(n); }
    NB_HD u32 cols() const { return ncols; }
    NB_HD const i32 *row(u64 r) const { return a + r * n; }
    // The A registers of k-step ks for rows g (row[0]) and g + 8 (row[1]) of a tile: mask words i0, i0 + 1 feed half 0,
    // i0 + 2, i0 + 3 half 1.  A row past the batch, and a word past n, is zero.
    NB_HD void a_frag(const i32 *const row[2], const bool ok[2], u32 ks, int t, u32 af[4]) const
    {
        const u32 i0 = 16 * ks + 4 * t;
        i32 w[2][4];
#pragma unroll
        for (int hr = 0; hr < 2; hr++)
#pragma unroll
            for (int q = 0; q < 4; q++) w[hr][q] = (ok[hr] && i0 + q < n) ? ldg(row[hr] + i0 + q) : 0;
        af[0] = tree_a_frag(w[0][0], w[0][1]);
        af[1] = tree_a_frag(w[1][0], w[1][1]);
        af[2] = tree_a_frag(w[0][2], w[0][3]);
        af[3] = tree_a_frag(w[1][2], w[1][3]);
    }
    NB_HD void store(u64 row, u32 col, u32 v, i32) const { out[row * ncols + col] = (i32)v; }
};

// ---- assembly
NB_HD int tree_box(int bits) { return PACK_N >> bits; }
// o_m = m box - box / 2: box m of the phase starts at o_m
NB_HD int tree_offset(int m, int bits) { return m * tree_box(bits) - tree_box(bits) / 2; }

// coefficient x of G_m,u: -V_u, plus the LWE body b at X^0 of the body polynomial (u = k)
NB_HD u32 tree_glwe_coef(const i32 *v_u, i32 b, bool body, int x)
{
    return (body && x == 0 ? (u32)b : 0u) - (u32)v_u[x];
}

// coefficient x of X^o * g, o in (-2N, 2N), is g[d] for d = (x - o) mod 2N < N, else -g[d - N]: the index into g and
// whether the value is negated
NB_HD int tree_shift_index(int o, int x, bool *neg)
{
    const int d = ((x - o) % (2 * PACK_N) + 2 * PACK_N) % (2 * PACK_N);
    *neg = d >= PACK_N;
    return d < PACK_N ? d : d - PACK_N;
}

// coefficient x of Q * z, Q = sum_{t < box} X^t, from the prefix sums ps[y] = z_0 + ... + z_{y-1}, y = 0 .. N.
// The negacyclic extension h of z (h[y + N] = -h[y]) sums to zero over 2N, so its prefix sums P(y) are 2N-periodic:
// P(y) = ps[y] for y <= N and ps[N] - ps[y - N] above; coefficient x is P(x + 1) - P(x + 1 - box).
NB_HD u32 tree_window_coef(const u32 *ps, int box, int x)
{
    const int lo = x + 1 - box;
    if (lo >= 0) return ps[x + 1] - ps[lo];
    return ps[x + 1] - ps[PACK_N] + ps[PACK_N + lo];
}

}  // namespace nb
