// mk_expand_layout.cuh -- where the multi-key expansion of compressed cloud keys (DESIGN.md section 19) reads and writes,
// kept apart from the kernels so that g++ compiles it into the host emulator (host_emul.cpp) and the CPU suite checks it
// against the ChaCha20 reference and the decompress() layout:
//   * nb_mk_bk_expand: the masks of the bootstrap key are the stream (seed, nonce 1) laid out (n, k+1, l, k, N), the
//     bodies are (n, k+1, l, N) int32; mask polynomial (i, mi, j, mo) is N consecutive words, N / 16 whole ChaCha blocks.
//     A CTA of 64 threads computes one block per thread and regroups the 1024 words through shared memory into the
//     stride-64 order bk_spectra_kernel reads (thread n0 holds coefficients 64 jj + n0, jj < 16);
//   * nb_mk_ks_expand: the masks of the key-switch key are the stream (seed, nonce 2) laid out (in, t, base-1, n); they
//     fill rows h = 1 .. base-1 of ks_a (in, t, base, n), whose rows h = 0 are zero.
#pragma once
#include "ff.cuh"

namespace nb {

// the nonces of the two mask streams (compressed.py: NONCE_BOOTSTRAP_KEY, NONCE_KEYSWITCH_KEY)
constexpr u64 MK_NONCE_BK = 1, MK_NONCE_KS = 2;

// stream word of coefficient 0 of mask polynomial (i, mi, j, mo < k) of the bootstrap key
NB_HD u64 mk_bk_mask_word(u64 i, u32 mi, u32 j, u32 mo, u32 k, u32 l, u32 N)
{
    return (((i * (k + 1) + mi) * l + j) * k + mo) * N;
}
// int32 offset of body polynomial (i, mi, j) in the bodies (n, k+1, l, N)
NB_HD u64 mk_bk_body_offset(u64 i, u32 mi, u32 j, u32 k, u32 l, u32 N) { return ((i * (k + 1) + mi) * l + j) * N; }

// The regrouping buffer: coefficient c = 16 b + w (word w of block b, written by thread b) sits at shared word
// mk_regroup_slot(c).  One pad word per block keeps the 32 lanes of a warp in distinct banks when each writes word w
// of its own block.
constexpr int MK_REGROUP_WORDS = 1024 + 64;
NB_HD int mk_regroup_slot(int c) { return c + (c >> 4); }
// the coefficient thread n0 reads at step jj (bk_spectra_kernel's order)
NB_HD int mk_spectra_coef(int n0, int jj) { return 64 * jj + n0; }

// word of ks_a (in, t, base, n) that stream word w of the key-switch masks (in, t, base-1, n) goes to: one zero row
// h = 0 precedes every base-1 mask rows
NB_HD u64 mk_ks_a_word(u64 w, u64 n, u32 base) { return w + (w / (n * (base - 1)) + 1) * n; }
// word of ks_a of coefficient c of zero row r (r < in t): row (r, h = 0)
NB_HD u64 mk_ks_zero_word(u64 r, u64 c, u64 n, u32 base) { return r * base * n + c; }

}  // namespace nb
