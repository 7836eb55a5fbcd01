// lut_index.cuh -- index functions of the programmable bootstrap (kernels.cuh, blind_rotate_kernel<Cfg, true>): the
// rounded mod-switch, the initial accumulator X^(2N - barb) * tv and the extraction of sample j.  Compiled by nvcc for
// the kernels and by g++ into the host emulator (host_emul.cpp), so the CPU suite checks the same code.
#pragma once
#include "ntt_lane.cuh"

namespace nb {

// mod-switch to [0, 2N), rounded to a multiple of 2^L: t32_to_phase with a message space of 2N / 2^L, times 2^L
// (numeric_functions_gpu.py:55-71).  L = 0 is the gate path's modswitch_2n.
NB_HD i32 modswitch_lut(i32 x, int L) { return (i32)((((u32)x + (1u << (20 + L))) >> (21 + L)) << L); }

// coefficient x of X^(2N - barb) * tv, barb in [0, 2N): the test vector rotated by -barb in the negacyclic ring
// (shift_tp_inverted_power, polynomials_gpu.mako:18-77); the sign rule of the gate path's constant test vector
NB_HD i32 lut_head_coef(const i32 *tv, int barb, int x)
{
    const int q = 2 * NTT_N - barb;
    if (q < NTT_N) return x < q ? (i32)(0u - (u32)tv[x + NTT_N - q]) : tv[x - q];
    return x < q - NTT_N ? tv[x + 2 * NTT_N - q] : (i32)(0u - (u32)tv[x + NTT_N - q]);
}

// mask coefficient x of the sample extracted at index j from the accumulator's mask polynomial a0: the extraction
// at index 0 after a rotation by X^(-j) (tlwe_gpu.mako:63-82).  The body is a1[j].
NB_HD i32 lut_tail_a(const i32 *a0, int j, int x) { return x <= j ? a0[j - x] : (i32)(0u - (u32)a0[NTT_N + j - x]); }

}  // namespace nb
