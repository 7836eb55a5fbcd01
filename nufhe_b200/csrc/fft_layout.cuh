// fft_layout.cuh -- where the FP64 CMux step (br_phases.cuh: FP64 step) keeps its spectra in shared memory, which
// positions each thread of the 2-ciphertext CTA (BrFft: 256 threads) reads and writes in each pass, and where the key
// spectra sit in an engine key row.  Compiled by nvcc for the kernels and by g++ into the host emulator
// (host_emul.cpp), so the CPU suite enumerates the 16-byte shared-memory accesses of every pass with the very functions
// the kernel uses and checks them for bank conflicts (tests/test_host_fft_layout.py).
#pragma once
#include "ntt_lane.cuh"

namespace nb {

constexpr int FFT_M = 512;                          // complex points per spectrum
constexpr int FFT_CT = 2;                           // ciphertexts per CTA of the FP64 step
// Position x (< 512) of a spectrum is stored at fft_pad(x) = x + x / 64 (one pad per 64), and the spectra are
// interleaved by ciphertext, [s][ct], at a stride of 522 = 2 mod 8 complex values.  One 16-byte access per thread
// touches bank group (offset mod 8); inside every quarter warp (8 lanes, one 128-byte wavefront) these all differ:
//   pass 1 (fwd1 / inv1): 8 consecutive n0 at x = n0 + 64 k          -> x mod 8 runs over 0..7;
//   pass 2: 8 blocks k1 at x = 64 k1 + n2 + 4 m (stride 4 inside)     -> the x / 64 term runs over 0..7;
//   pass 3: groups g0 + {0, 1, 16, 17} at x = 4 g + i, 2 ciphertexts  -> 4 g + g / 16 takes c + {0, 4, 1, 5}, and the
//           second ciphertext, 2 mod 8 further on, c + {2, 6, 3, 7} (fft_pass3_group).
// Every address of a pass is then a per-thread base plus a compile-time offset.
constexpr int FFT_SPEC_CPLX = 522;                  // >= fft_pad(511) + 1 = 519, and 2 mod 8
NB_HD int fft_pad(int x) { return x + (x >> 6); }
// spectrum s (0..3) of ciphertext ct of the CTA, interleaved [s][ct]
NB_HD int fft_spec(int ct, int s) { return (s * FFT_CT + ct) * FFT_SPEC_CPLX; }

// pass 1 (fwd1 / inv1): thread tid = (pm = ct * 2 + poly, n0): positions n0 + 64 k (k < 8) of spectra poly * 2 + h,
// h = 0, 1 (fwd1: the two digits of accumulator polynomial poly = mi; inv1: the two key halves of output polynomial
// poly = mo)
NB_HD int fft_pass1_spec(int tid, int h) { return fft_spec(tid >> 7, ((tid >> 6) & 1) * 2 + h); }
NB_HD int fft_pass1_x(int n0, int k) { return fft_pad(n0 + 64 * k); }          // stored position inside a spectrum
NB_HD int fft_pass1_pos(int tid, int h, int k) { return fft_pass1_spec(tid, h) + fft_pass1_x(tid & 63, k); }
// pass 2 (fwd2 / inv2): warp = (ct, n2), lane = (s, k1): the 16 positions 64 k1 + n2 + 4 m of spectrum s.  n2 is
// warp-uniform, so every twiddle load W64^(n2 k2) of a warp-instruction reads one address.
struct FftPass2 {
    int ct, s, k1, n2;
};
NB_HD FftPass2 fft_pass2_task(int tid) { return {tid >> 7, (tid >> 3) & 3, tid & 7, (tid >> 5) & 3}; }
NB_HD int fft_pass2_x(int k1, int n2, int m) { return fft_pad(64 * k1 + n2 + 4 * m); }
NB_HD int fft_pass2_pos(const FftPass2 &t, int m) { return fft_spec(t.ct, t.s) + fft_pass2_x(t.k1, t.n2, m); }
// pass 3 (fused DFT4, MAC, inverse DFT4): thread tid = (j = tid / 2, ct = tid & 1) works on group g = fft_pass3_group(j)
// (g = 16 k1 + k2): the 4 positions 4 g + i of each spectrum s of ciphertext ct.  Both ciphertexts of a group sit on
// adjacent lanes, so one key load serves both; the 4 groups of a quarter warp are g0 + {0, 1, 16, 17} (bit 1 of j is
// bit 4 of g), which spreads them over the bank groups.
NB_HD int fft_pass3_group(int j) { return (j & 1) | (((j >> 1) & 1) << 4) | (((j >> 2) & 7) << 1) | ((j >> 5) << 5); }
NB_HD int fft_pass3_x(int g, int i) { return fft_pad(4 * g + i); }
NB_HD int fft_pass3_pos(int tid, int s, int i) { return fft_spec(tid & 1, s) + fft_pass3_x(fft_pass3_group(tid >> 1), i); }

// Key spectra of an engine key row (the FP64 part, BK_FFT_U64): 16 spectra ks = (m = (mi * 2 + j) * 2 + mo) * 2 + h,
// each stored [k3][j]: the point that pass 3 computes as output k3 of group fft_pass3_group(j).  The 16 thread pairs
// of a warp read 256 contiguous bytes per key load.
NB_HD int fft_key_pos(int ks, int j, int k3) { return ks * FFT_M + k3 * (FFT_M / 4) + j; }

}  // namespace nb
