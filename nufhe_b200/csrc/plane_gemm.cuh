// plane_gemm.cuh -- the exact 32-bit integer GEMM on the tensor cores that public-key encryption (DESIGN.md section 11)
// and the tree key switch (section 13) share, kept apart from the MMA so that g++ compiles it into the host emulator
// (host_emul.cpp) and the CPU suite checks it:
//   * the byte-plane layout the prepare kernel writes,
//   * which plane bytes each lane feeds to the m16n8k32 B fragments,
//   * the row and column of each accumulator in the epilogue, and the recombination of the four plane sums,
//   * the bound that keeps every s32 accumulator exact.
// The product is OUT (rows x cols) = A (rows x K) x W (K x cols) mod 2^32.  W is split once into 4 byte planes
// W = sum_p 2^(8p) W_p; each plane product is an exact 8-bit x u8 -> s32 GEMM, and an output word is
// S0 + 2^8 S1 + 2^16 S2 + 2^24 S3 mod 2^32.  What A is, and what becomes of an output word, is the caller's operand
// policy (PkGemm in pk_layout.cuh, TreeGemm in tree_layout.cuh).
#pragma once
#include "ff.cuh"

namespace nb {

constexpr int GEMM_WARPS = 4;     // warps per CTA: each its own 64-row slice, all on the same NTILES * 8 columns
constexpr int GEMM_MTILES = 4;    // m16 tiles per warp (64 rows)

// Plane p is column-major K x cols (the `.col` B operand): byte (k, col) at ((p * cols + col) * K + k).
NB_HD u64 plane_offset(u32 p, u32 col, u32 k, u32 K, u32 cols) { return ((u64)p * cols + col) * K + k; }

// The four K values a lane with threadID_in_group t feeds to fragment half h of a k-step: h = 0 is registers a0/a1
// and b0, h = 1 is a2/a3 and b1 (the PTX ISA's logical k offset of 16).  The kernel is free to choose which actual K
// values sit in which logical slot, as long as A and B agree: this order lets each lane read 8 consecutive plane
// bytes per column and 8 consecutive K values of A per row.
NB_HD u32 frag_k(int t, int h) { return 8 * t + 4 * h; }

// Accumulator register i (0..3) of lane (groupID g, threadID_in_group t): row g (+8 for i >= 2), column 2t + (i & 1).
NB_HD u32 acc_row(int g, int i) { return g + 8 * (i >> 1); }
NB_HD u32 acc_col(int t, int i) { return 2 * t + (i & 1); }

// The output word of the four plane sums of one (row, column).
NB_HD u32 combine(i32 s0, i32 s1, i32 s2, i32 s3)
{
    return (u32)s0 + ((u32)s1 << 8) + ((u32)s2 << 16) + ((u32)s3 << 24);
}

// Every plane sum is at most K * max|A byte| * 255; the s32 accumulators are exact while that is below 2^31.
NB_HD bool plane_gemm_exact(u64 K, u32 max_a) { return K <= ((1ull << 31) - 1) / (255ull * max_a); }

// A global load through the read-only cache on the device, a plain load in the host emulator.
template <class T> NB_HD T ldg(const T *p)
{
#if defined(__CUDA_ARCH__)
    return __ldg(p);
#else
    return *p;
#endif
}

}  // namespace nb
