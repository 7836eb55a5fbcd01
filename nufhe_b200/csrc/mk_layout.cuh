// mk_layout.cuh -- the tables of the multi-key tree key switch and packing MAC (DESIGN.md section 18), kept apart from
// the kernels so that g++ compiles them into the host emulator (host_emul.cpp) and the CPU suite checks them:
//   * nb_mk_tree_keyswitch: the batch is counts[0] rows of tenant 0, then counts[1] rows of tenant 1, ...; CTA x of the
//     byte-plane GEMM takes tile x, up to MK_TILE_ROWS consecutive rows of ONE tenant with that tenant's planes, so a
//     tile never crosses a tenant boundary and every row lies in exactly one tile;
//   * nb_mk_ntt_mac: group_counts[t] consecutive groups belong to tenant t; group g reads the key spectra of its tenant.
#pragma once
#include <stddef.h>
#include "plane_gemm.cuh"

namespace nb {

constexpr u32 MK_TILE_ROWS = GEMM_WARPS * GEMM_MTILES * 16;      // the rows of one CTA of plane_gemm_kernel: 256

struct TreeTile {
    const uint8_t *planes;      // the tenant's nb_tree_prepare planes
    u64 row0;                   // first row of the batch
    u32 rows;                   // 1 .. MK_TILE_ROWS
    u32 tenant;
};

// The tiles of `counts` (tenants entries), written to `out` unless it is null; returns their number.
inline u64 mk_tree_tiles(const size_t *counts, size_t tenants, const uint8_t *const *planes, TreeTile *out)
{
    u64 n = 0, row = 0;
    for (size_t t = 0; t < tenants; row += counts[t], t++)
        for (u64 q = 0; q < counts[t]; q += MK_TILE_ROWS, n++)
            if (out) {
                const u64 left = counts[t] - q;
                out[n] = {planes ? planes[t] : nullptr, row + q, (u32)(left < MK_TILE_ROWS ? left : MK_TILE_ROWS), (u32)t};
            }
    return n;
}

// The key of every group: out[g] = keys[t] for the tenant t that owns group g.  Returns the number of groups.
template <class K> inline u64 mk_group_keys(const size_t *group_counts, size_t tenants, const K *keys, K *out)
{
    u64 g = 0;
    for (size_t t = 0; t < tenants; t++)
        for (size_t i = 0; i < group_counts[t]; i++, g++)
            if (out) out[g] = keys[t];
    return g;
}

}  // namespace nb
