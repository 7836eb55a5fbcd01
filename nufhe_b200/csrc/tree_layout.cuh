// tree_layout.cuh -- the index and sign arithmetic of tree-based programmable bootstrapping (DESIGN.md section 13),
// kept apart from the kernels so that g++ compiles it into the host emulator (host_emul.cpp) and the CPU suite checks
// it:
//   * the LWE -> GLWE key switch V (R, k+1, N) = D (R, n t) x T (n t, (k+1) N) mod 2^32 as an exact byte-plane GEMM:
//     the plane layout nb_tree_prepare writes, the signed 8-bit digit fragments a lane forms from two mask words, and
//     the row / column of each accumulator (the m16n8k32 fragment layout is the one of pk_layout.cuh);
//   * the test-vector assembly tv_u = sum_m X^(o_m) Q_P G_m,u (negacyclic) with Q_P = 1 + X + ... + X^(box - 1):
//     Z_u = sum_m X^(o_m) G_m,u first, then the box sum of Z_u from its prefix sums.
#pragma once
#include "pack_layout.cuh"
#include "pk_layout.cuh"

namespace nb {

constexpr int TREE_WARPS = 4;     // warps per CTA, each its own 64-row slice, all on the same TREE_NTILES * 8 columns
constexpr int TREE_MTILES = 4;    // m16 tiles per warp
constexpr int TREE_NTILES = 2;    // n8 tiles per CTA

// digit rows n t padded to whole k-steps of 32 (the padding rows of the key planes are zero)
NB_HD u32 tree_k_padded(u32 n) { return (n * PACK_LEVELS + 31u) & ~31u; }

// Plane p is column-major kpad x cols (the `.col` B operand): byte (kk, col) at ((p * cols + col) * kpad + kk).
NB_HD u64 tree_plane_offset(u32 p, u32 col, u32 kk, u32 kpad, u32 cols) { return ((u64)p * cols + col) * kpad + kk; }

// T[kk][col], kk = i t + j, col = u N + x: mask u < k of key row kk (masks (n, t, k, N)) or its body (bodies (n, t, N))
NB_HD u32 tree_key_word(const i32 *masks, const i32 *body, u32 n, u32 k, u32 kk, u32 col)
{
    if (kk >= n * PACK_LEVELS) return 0u;
    const u32 u = col / PACK_N, x = col % PACK_N;
    return u < k ? (u32)masks[((u64)kk * k + u) * PACK_N + x] : (u32)body[(u64)kk * PACK_N + x];
}

// The A fragment register of K values kb .. kb + 3 (kb = 32 ks + pk_frag_k(t, h), even): the digits d_0, d_1 of mask
// words kb / 2 and kb / 2 + 1 as four signed bytes, lowest first.  Byte 3 - j of pack_digit_word is d_j + 128, so the
// signed byte is that byte with its top bit flipped.
NB_HD u32 tree_a_frag(i32 a0, i32 a1)
{
    const u32 w0 = pack_digit_word(a0), w1 = pack_digit_word(a1);
    const u32 v = (w0 >> 24) | (((w0 >> 16) & 0xFFu) << 8) | ((w1 >> 24) << 16) | (((w1 >> 16) & 0xFFu) << 24);
    return v ^ 0x80808080u;
}

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
