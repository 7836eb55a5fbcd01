"""The layouts of the multi-key entry points (nb_mk_*, DESIGN.md sections 17 and 18) and the oracle compositions of
their bootstraps, for the multi-key matrix (tests/test_gpu_multikey_matrix.py).  TEST INFRASTRUCTURE ONLY; it shares
no code with the CUDA source.

The layout rules restate nufhe_b200/csrc/capi.cu and csrc/mk_layout.cuh as functions of the tenant counts (and, for
the key switch, of the registered tenants, the engine's GEMM threshold and the SM count); nothing in the library is
configured from here, so if those files change their rules this file must follow them."""
import types

import numpy

import fused_ref as F
import ks_ref as K

KS_TILE = 32            # rows of one gather tile of nb_mk_keyswitch (kernels.cuh: KS_TILE)
KS_MAX_SPLITS = 128
TREE_TILE = 256         # rows of one tile of nb_mk_tree_keyswitch (mk_layout.cuh: MK_TILE_ROWS)
BR_CT, BR_CTAS_PER_SM = 2, 2     # BrFftMk: ciphertexts per CTA, CTAs per SM


def tenant_of(counts, jobs=1):
    """the tenant that owns every row: counts[0] rows of tenant 0, then counts[1] of tenant 1, ...; with `jobs` jobs
    (extract2: 2) the batch is repeated once per job, rows of job j at [j B, (j + 1) B)"""
    one = numpy.repeat(numpy.arange(len(counts)), numpy.asarray(counts, numpy.int64))
    return numpy.tile(one, jobs)


def segments(counts):
    """(tenant, first row, end row) of every tenant"""
    lo = 0
    for t, c in enumerate(counts):
        yield t, lo, lo + int(c)
        lo += int(c)


def truncate(counts, B):
    """the first B rows of a layout: the tenant that holds row B - 1 keeps the rows up to it, the tenants after it
    become idle (count 0), so the tenant list stays the same"""
    out, left = [], B
    for c in counts:
        out.append(min(int(c), left))
        left -= out[-1]
    assert left == 0, (B, sum(counts))
    return out


def wave(sm_count):
    """ciphertexts in one wave of resident BrFftMk CTAs"""
    return BR_CT * BR_CTAS_PER_SM * sm_count


# ---- the bootstraps, per tenant -------------------------------------------------------------------------------------

def _sub(x, idx):
    return None if x is None else (numpy.asarray(x[0])[idx], numpy.asarray(x[1])[idx])


def ref(owner):
    """the compositions of fused_ref's modes for a multi-key batch: `owner` is the tenant of each selected row (job rows
    for extract2, whose two jobs have the same owners), and the key argument `bk` is the sequence of every tenant's key
    in the reference's form.  Each tenant's rows go through fused_ref.STANDARD with that tenant's key (in one call for
    all the tenants that share one key object)."""
    owner = numpy.asarray(owner)

    def split(call, per_row, bk):
        out_a = out_b = None
        groups = {}
        for t in numpy.unique(owner):
            groups.setdefault(id(bk[t]), (int(t), []))[1].append(t)
        for t, ts in groups.values():
            idx = numpy.flatnonzero(numpy.isin(owner, ts))
            a, b = call(idx, t)
            a, b = numpy.asarray(a), numpy.asarray(b)
            if out_a is None:
                out_a = numpy.empty((owner.size, per_row, a.shape[-1]), numpy.int32)
                out_b = numpy.empty((owner.size, per_row), numpy.int32)
            out_a[idx] = a.reshape(idx.size, per_row, -1)
            out_b[idx] = b.reshape(idx.size, per_row)
        return out_a.reshape(owner.size * per_row, -1), out_b.reshape(-1)

    def bootstrap_extract(x1, x2, c, s1, s2, mu, bk):
        return split(lambda idx, t: F.STANDARD.bootstrap_extract(_sub(x1, idx), _sub(x2, idx), c, s1, s2, mu, bk[t]),
                     1, bk)

    def bootstrap_lut_extract(x1, x2, c, s1, s2, tv, L, bk):
        tv = numpy.asarray(tv)
        return split(lambda idx, t: F.STANDARD.bootstrap_lut_extract(_sub(x1, idx), _sub(x2, idx), c, s1, s2,
                                                                     tv if tv.ndim == 1 else tv[idx], L, bk[t]),
                     1 << L, bk)

    def bootstrap_glwe_lut_extract(x, tv, bk):
        tv = numpy.asarray(tv)
        return split(lambda idx, t: F.STANDARD.bootstrap_glwe_lut_extract(_sub(x, idx), tv[idx], bk[t]), 1, bk)

    return types.SimpleNamespace(bootstrap_extract=bootstrap_extract, bootstrap_lut_extract=bootstrap_lut_extract,
                                 bootstrap_glwe_lut_extract=bootstrap_glwe_lut_extract)


# ---- nb_mk_keyswitch's dispatch (capi.cu) ---------------------------------------------------------------------------

def ks_gemm_tenants(counts, registered, ks_mma_min):
    """the tenants whose segment runs as the tensor-core GEMM (nb_keyswitch on that segment): a registered key and at
    least ks_mma_min rows (the rows of the matrix are 16-byte aligned, so the alignment rule never declines one)"""
    return [t for t, c in enumerate(counts) if c and t in registered and c >= ks_mma_min]


def ks_tiles(counts, registered=(), ks_mma_min=None):
    """[(tenant, first row, rows)] of keyswitch_grouped_kernel: every other tenant's rows in tiles of up to 32, which
    never cross a tenant"""
    gemm = set(ks_gemm_tenants(counts, registered, ks_mma_min)) if registered else set()
    return [(t, lo + q, min(KS_TILE, hi - lo - q)) for t, lo, hi in segments(counts) if t not in gemm
            for q in range(0, hi - lo, KS_TILE)]


def ks_splits(tiles, sm_count):
    """the j split of the gather launch: min(128, SMs / tiles), at least 1"""
    return max(1, min(KS_MAX_SPLITS, sm_count // tiles))


def ks_split_bands(sm_count):
    """{splits: (first tile count, last tile count)}, the band of one split open (last None): ks_ref.gather_bands, whose
    rule over the grid of a single-key launch is the same rule over tiles"""
    return K.gather_bands(sm_count)


KS_PATTERN = (1, 31, 32, 33, 5, 17)      # tenant counts the band builder cycles through (1 or 2 tiles each)


def ks_counts_with_tiles(tiles):
    """a gather-only count list with exactly `tiles` tiles: tenants cycle through KS_PATTERN (segments of 31, 32 and 33
    rows, partial tiles) while they fit, then ones"""
    counts, left, i = [], tiles, 0
    while left:
        c = KS_PATTERN[i % len(KS_PATTERN)]
        need = -(-c // KS_TILE)
        if need > left:
            c, need = 1, 1
        counts.append(c)
        left -= need
        i += 1
    return counts


def ks_band_mixes(sm_count):
    """[(splits, counts)]: the first and the last tile count of every split band (the open band: its first two)"""
    out = []
    for s, (lo, hi) in sorted(ks_split_bands(sm_count).items()):
        for tiles in sorted({lo, hi if hi is not None else lo + 1}):
            out.append((s, ks_counts_with_tiles(tiles)))
    return out


# ---- nb_mk_tree_keyswitch and nb_mk_ntt_mac (mk_layout.cuh) --------------------------------------------------------

def tree_tiles(counts):
    """[(first row, rows, tenant)] of tree_gemm_mk_kernel: up to 256 consecutive rows of one tenant per tile"""
    return [(lo + q, min(TREE_TILE, hi - lo - q), t) for t, lo, hi in segments(counts)
            for q in range(0, hi - lo, TREE_TILE)]


def group_tenants(group_counts):
    """the tenant of every group of nb_mk_ntt_mac, whose key spectra the group reads"""
    return tenant_of(group_counts)
