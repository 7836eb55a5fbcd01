"""Host-side model of nb_keyswitch's launch shapes and of its fixed-shape variance sum, and builders of edge inputs and
edge keys for the key-switch matrix (tests/test_gpu_keyswitch_matrix.py).  TEST INFRASTRUCTURE ONLY.

The launch rules restate nb_keyswitch in nufhe_b200/csrc/capi.cu as functions of (batch, SM count); nothing in the
library is configured from here, so if capi.cu changes its rules this file must follow it."""
import numpy

import ks_mma_ref as R

IN, T, BASE, N_OUT = 1024, 8, 4, 500
KS_TILE = 32            # kernels.cuh: ciphertexts per CTA of keyswitch_kernel
CV_BLOCK_J = 8          # kernels.cuh: KS_CV_BLOCK_J, input coefficients per variance block
CV_BLOCKS = IN // CV_BLOCK_J
KM_M, KM_NTILES = 256, 16   # kernels.cuh: ciphertexts per CTA and N tiles of keyswitch_mma_kernel
KM_MAX_SPLITS = 16


# ---- launch shapes (capi.cu, nb_keyswitch) --------------------------------------------------------------------------

def gather_launch(batch, sm_count):
    """(tile, grid, splits, j_per) of keyswitch_kernel: tiles of up to 32 ciphertexts, then the 1024 input coefficients
    split over blockIdx.y while the SMs are not covered; each split takes j_per coefficients, a multiple of 8"""
    tile = min(batch, KS_TILE)
    grid = -(-batch // tile)
    splits = max(1, min(128, sm_count // grid))
    return tile, grid, splits, j_per(splits)


def j_per(splits):
    return (-(-IN // splits) + CV_BLOCK_J - 1) // CV_BLOCK_J * CV_BLOCK_J


def j_slices(splits):
    """[(j_begin, j_end)] of blockIdx.y = 0 .. splits - 1 (trailing slices may be empty)"""
    p = j_per(splits)
    return [(min(IN, y * p), min(IN, (y + 1) * p)) for y in range(splits)]


def mma_launch(batch, sm_count):
    """(M tiles, CTAs per K slice, splits) of keyswitch_mma_kernel: K is halved while the launch would leave half of
    the SMs idle, up to 16 ways"""
    m_tiles = -(-batch // KM_M)
    tiles = m_tiles * KM_NTILES
    splits = 1
    while splits < KM_MAX_SPLITS and tiles * splits * 2 <= sm_count:
        splits *= 2
    return m_tiles, tiles, splits


def gather_bands(sm_count):
    """{splits: (first grid, last grid)} of keyswitch_kernel; the band of splits = 1 is open, its last grid is None"""
    bands = {}
    g = 1
    while True:
        s = gather_launch(KS_TILE * g, sm_count)[2]
        lo, hi = bands.get(s, (g, g))
        bands[s] = (lo, g)
        if s == 1:
            bands[1] = (lo, None)
            return bands
        g += 1


def mma_bands(sm_count):
    """{splits: (first batch, last batch)} of keyswitch_mma_kernel; the band of splits = 1 is open (last None)"""
    bands = {}
    m = 1
    while True:
        s = mma_launch(KM_M * m, sm_count)[2]
        lo, _ = bands.get(s, (KM_M * (m - 1) + 1, None))
        bands[s] = (lo, KM_M * m)
        if s == 1:
            bands[1] = (lo, None)
            return bands
        m += 1


def gather_batches(sm_count):
    """{splits: batches}: the first and the last batch of each split band of keyswitch_kernel (32 g - 31 at its
    first grid g, 32 g at its last); the open band of one split gets its first two edges"""
    out = {}
    for s, (lo, hi) in gather_bands(sm_count).items():
        out[s] = sorted({KS_TILE * lo - (KS_TILE - 1), KS_TILE * (hi if hi is not None else lo)})
    return out


def mma_batches(sm_count):
    """{splits: batches}: the first and the last batch of each split band of keyswitch_mma_kernel (the open band of one
    split: its first batch)"""
    return {s: sorted({lo, hi if hi is not None else lo}) for s, (lo, hi) in mma_bands(sm_count).items()}


MULTI_WAVE = (4097, 16384)


def matrix_batches(sm_count):
    """every batch the matrix runs: the band edges of both fast paths, 1 and 256, and multi-wave batches"""
    bs = {1, KM_M} | set(MULTI_WAVE)
    for d in (gather_batches(sm_count), mma_batches(sm_count)):
        for v in d.values():
            bs |= set(v)
    return sorted(bs)


# ---- the fixed-shape float32 variance (kernels.cuh: KS_CV_BLOCK_J) -------------------------------------------------

def variance(ks_cv, src_a):
    """(B,) float32 variances as the fast kernels add them: 128 block sums of 8 coefficients x 8 digits, each added in
    (j, k) order from 0, then the block sums added in block order from 0"""
    ks_cv = numpy.asarray(ks_cv, numpy.float32).reshape(IN, T, BASE)
    d = R.digits(numpy.asarray(src_a, numpy.int32)).astype(numpy.intp)           # (B, 1024, 8)
    terms = ks_cv[numpy.arange(IN)[:, None], numpy.arange(T)[None, :], d]          # (B, 1024, 8) float32
    terms = terms.reshape(terms.shape[0], CV_BLOCKS, CV_BLOCK_J * T)
    blk = numpy.zeros(terms.shape[:2], numpy.float32)
    for i in range(CV_BLOCK_J * T):
        blk += terms[:, :, i]
    cv = numpy.zeros(terms.shape[0], numpy.float32)
    for b in range(CV_BLOCKS):
        cv += blk[:, b]
    return cv


# additions on one path from a term to the result: 63 inside its block, 127 over the block sums
VARIANCE_ADDS = CV_BLOCK_J * T - 1 + CV_BLOCKS - 1


def variance_f64(ks_cv, src_a):
    """(sum of the terms, sum of their magnitudes) in float64, for the error bound of `variance`"""
    ks_cv = numpy.asarray(ks_cv, numpy.float32).reshape(IN, T, BASE).astype(numpy.float64)
    d = R.digits(numpy.asarray(src_a, numpy.int32)).astype(numpy.intp)
    terms = ks_cv[numpy.arange(IN)[:, None], numpy.arange(T)[None, :], d]
    return terms.sum(axis=(1, 2)), numpy.abs(terms).sum(axis=(1, 2))


# ---- edge inputs ---------------------------------------------------------------------------------------------------

def u32(x):
    return numpy.asarray(x, numpy.int64) & 0xFFFFFFFF


def i32(x):
    return u32(x).astype(numpy.uint32).view(numpy.int32)


ALL_THREE = 0xFFFF7FFF      # rounds to 0xFFFF: every digit 3
ALL_ZERO_WRAP = 0xFFFF8000  # the rounding carry leaves bit 31: every digit 0


def edge_coefficients():
    """[(uint32 coefficient, its 8 digits)]: the two rounding-carry edges, and each digit value 1..3 alone in each of
    the 8 positions at the lowest and the highest coefficient that rounds to it"""
    out = [(ALL_THREE, [3] * T), (ALL_ZERO_WRAP, [0] * T), (0, [0] * T), (0x7FFF, [0] * T)]
    for k in range(T):
        for v in (1, 2, 3):
            word = v << (14 - 2 * k)
            dg = [0] * T
            dg[k] = v
            out.append((((word << 16) - (1 << 15)) & 0xFFFFFFFF, dg))
            out.append((((word << 16) + (1 << 15) - 1) & 0xFFFFFFFF, dg))
    return out


def edge_rows(rng, B):
    """(B, 1024) int32 inputs: row 0 all digits 3, row 1 wraps to all digits 0, the next rows cycle the edge
    coefficients over j at a different offset each, the rest random"""
    coeffs = numpy.array([c for c, _ in edge_coefficients()], numpy.int64)
    src = rng.randint(-2**31, 2**31, size=(B, IN), dtype=numpy.int64)
    if B > 0:
        src[0] = ALL_THREE
    if B > 1:
        src[1] = ALL_ZERO_WRAP
    for r in range(2, min(B, 2 + coeffs.size)):
        src[r] = numpy.roll(numpy.resize(coeffs, IN), r - 2)
    return i32(src)


def fold_pair(rng, target):
    """(src1, src2) int32 with src1 + src2 = target mod 2^32 and a carry out of bit 31 (the sum wraps), except for the
    target 2^32 - 1, which no pair of 32-bit words reaches with a carry"""
    t = u32(target)
    span = 0xFFFFFFFF - t
    r = rng.randint(0, 2**62, size=t.shape, dtype=numpy.int64)
    s1 = numpy.where(span > 0, t + 1 + r % numpy.maximum(span, 1), r & 0xFFFFFFFF)
    s2 = (t - s1) & 0xFFFFFFFF
    return i32(s1), i32(s2)


# ---- edge keys -----------------------------------------------------------------------------------------------------

KEY_KINDS = ('generated', 'random', 'bytes_ff', 'min_word', 'tagged')
TAG_MULT = 0x9E3779B1       # odd: a bijection of the 32-bit words


def tagged_key(in_size=IN, t=T, base=BASE, n=N_OUT):
    """(ks_a, ks_b, ks_cv) whose word at (j, k, d, x) is an odd multiple of the position's index (ks_b in column n), so
    any mix-up of rows or columns changes the result; rows d = 0 are zero, as in a generated key"""
    j, k, d, x = numpy.meshgrid(numpy.arange(in_size), numpy.arange(t), numpy.arange(base), numpy.arange(n + 1),
                                indexing='ij', sparse=True)
    tag = (((j * t + k) * base + d) * (n + 1) + x).astype(numpy.int64) + 1
    w = i32(tag * TAG_MULT)
    w[:, :, 0, :] = 0
    ks_a = numpy.ascontiguousarray(w[..., :n])
    ks_b = numpy.ascontiguousarray(w[..., n])
    ks_cv = ((tag[..., 0] % 1009).astype(numpy.float32) + 1) * numpy.float32(1e-9)
    return ks_a, ks_b, ks_cv


def edge_key(kind, rng):
    """a key-switch key (1024, 8, 4, 500) of `kind` (not 'generated', which is the oracle's key): random, every byte
    0xFF or every word -2^31, or tagged; rows d = 0 zero.  'pad' is random with non-zero d = 0 rows"""
    if kind == 'tagged':
        return tagged_key()
    ks_a = rng.randint(-2**31, 2**31, size=(IN, T, BASE, N_OUT), dtype=numpy.int32)
    ks_b = rng.randint(-2**31, 2**31, size=(IN, T, BASE), dtype=numpy.int32)
    ks_cv = rng.uniform(0.0, 1e-6, size=(IN, T, BASE)).astype(numpy.float32)
    if kind == 'bytes_ff':
        ks_a[:] = -1
        ks_b[:] = -1
    elif kind == 'min_word':
        ks_a[:] = -2**31
        ks_b[:] = -2**31
    else:
        assert kind in ('random', 'pad'), kind
    if kind != 'pad':
        ks_a[:, :, 0] = 0
        ks_b[:, :, 0] = 0
    return ks_a, ks_b, ks_cv
