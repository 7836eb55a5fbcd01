// compact_layout.cuh -- the index, rounding and extraction functions of compact public-key encryption (DESIGN.md
// section 16), kept apart from the kernels so that g++ compiles them into the host emulator (host_emul.cpp) and the
// CPU suite checks them:
//   * the slot mapping is packing's (pack_layout.cuh): message c (C order) goes to group c / N, slot c % N;
//   * one output coefficient of a compact ciphertext: the 32-bit sum (product + noise, plus the message on an
//     occupied body slot, or 0 on an empty body slot) rounded to 16 bits with packing's rounding;
//   * sample extraction of slot p from a restored GLWE sample: a'[u N + j] = A'_u[p - j] for j <= p and
//     -A'_u[N + p - j] for j > p, b' = body'[p] (tlwe_extract_lwe_samples is the case p = 0).
#pragma once
#include "pack_layout.cuh"

namespace nb {

// coefficient u N + j of a compact ciphertext's group: mask polynomial u < k, or the body u = k whose coefficient j is
// slot j.  `occupied`: slot j of this group holds a message (empty body slots are stored as 0).
NB_HD uint16_t compact_coeff(u32 product, u32 noise, bool body, bool occupied, u32 mu)
{
    if (body && !occupied) return 0;
    return pack_round16(product + noise + (body ? mu : 0u));
}

// the coefficient of A'_u that extracted mask word j of slot p reads, and whether it is negated
NB_HD u32 compact_extract_src(u32 p, u32 j) { return (p - j) & (u32)(PACK_N - 1); }
NB_HD bool compact_extract_negated(u32 p, u32 j) { return j > p; }

// extracted mask word j of slot p from the restored polynomial A' (N words, coefficients already shifted by 16 bits)
NB_HD i32 compact_extract(const u32 *a, u32 p, u32 j)
{
    const u32 v = a[compact_extract_src(p, j)];
    return (i32)(compact_extract_negated(p, j) ? 0u - v : v);
}

}  // namespace nb
