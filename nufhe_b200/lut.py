"""Programmable bootstrapping: lookup tables on small encrypted integers.

Encoding.  An integer ciphertext with a message space of P bits (P = 1, 2 or 3) holds m in [0, 2^P) as the Torus32
value m * 2^(31 - P).  The upper half of the torus is padding, so the negacyclic wrap of the blind rotation never mixes
two messages.  All integer ciphertexts of one computation share one P; smaller values, such as a bit, live in the same
space.

A bootstrap with test vector tv computes coefficient 0 of X^(-p) * tv, where p in [0, 2N) is the mod-switched phase.
`make_test_vector` lays a table f out so that this coefficient is f(m) for every phase in the box of m: box m is the
half-open range of width N / 2^P centred on m * N / 2^P.  The top half-box, reached by m = 0 with a negative error,
holds -f(0), which the wrap turns back into f(0).  With 2^L outputs the phase is rounded to a multiple of 2^L, output
i sits at the positions congruent to i mod 2^L, and coefficient j of the rotated vector -- extracted as sample j -- is
f_j(m) (the "many-LUT" technique: several functions of one input from one blind rotation).

A bivariate table packs two inputs as x * 2^shift + y before the bootstrap; the fused kernel forms that sum in its
prologue.  The noise of a LUT input decides which (P, L, shift) are safe (`check_noise`, DESIGN.md section 9).
"""
import numpy
import torch

from .numeric_functions import t32_to_phase
from .lwe import LweSampleArray
from .polynomials import TorusPolynomialArray, shift_tp_inverted_power
from .tlwe import TLweSampleArray, tlwe_noiseless_trivial, tlwe_extract_lwe_samples
from .bootstrap import blind_rotate
from .gates import MU, check_shape
from .batch_keys import OneKey

MAX_BITS = 3
MAX_LOG2_OUTPUTS = 2
MARGIN_SIGMAS = 7          # a LUT input must lie this many standard deviations inside its box

# (P, L, shift) the default parameter set allows; shift None = one input.  Follows from lut_sigma (tests check it).
# The measured noise rules out P = 3 and shift 1, which the estimates alone would allow (DESIGN.md section 9).
ALLOWED = {
    (1, 0, None), (1, 1, None), (1, 2, None), (1, 0, 0), (1, 1, 0), (1, 2, 0),
    (2, 0, None), (2, 1, None), (2, 0, 0), (2, 1, 0),
}

# Standard deviations (torus units) of the rounded input phase measured by tools/lut_noise.py for the default parameter
# set, keyed by (L, shift), over 65 536 inputs that are themselves LUT outputs, on an H100 80GB HBM3 (700 W, 1980 MHz)
# (DESIGN.md section 9).  All lie 3 - 13 % above the estimates; lut_sigma takes the larger of the two.
MEASURED_SIGMA = {
    (0, None): 0.00466, (0, 0): 0.00621, (0, 1): 0.00942,
    (1, None): 0.00607, (1, 0): 0.00732, (1, 1): 0.01018,
    (2, None): 0.00993, (2, 0): 0.01074, (2, 1): 0.01287,
}


def _check_bits(bits):
    if int(bits) != bits or not 1 <= bits <= MAX_BITS:
        raise ValueError("the message space must have 1 to %d bits, got %r" % (MAX_BITS, bits))


def encode_int(values, bits):
    """Torus32 encoding m * 2^(31 - bits) of integers m in [0, 2^bits)."""
    _check_bits(bits)
    values = numpy.asarray(values)
    if values.size and (values.min() < 0 or values.max() >= 2**bits):
        raise ValueError("values must lie in [0, %d)" % 2**bits)
    return (values.astype(numpy.int64) << (31 - bits)).astype(numpy.int32)


def decode_int(phases, bits):
    """The integer in [0, 2^bits) nearest to each Torus32 phase (a phase in the padding half decodes modulo 2^bits)."""
    _check_bits(bits)
    u = numpy.asarray(phases).astype(numpy.int64) & 0xffffffff
    return (((u + (1 << (30 - bits))) & 0xffffffff) >> (31 - bits)) % (1 << bits)


def make_test_vector(tables, bits, log2_outputs=0, out='int'):
    """Test vectors (..., 1024) int32 for `tables` of shape batch + (2^bits,) (L = 0) or batch + (2^L, 2^bits).
    out='int': output values are taken modulo 2^bits and encoded like the inputs; out='bool': nonzero entries give
    +gates.MU, zeros -gates.MU, so the results feed the gate_* functions."""
    _check_bits(bits)
    L = int(log2_outputs)
    if not 0 <= L <= MAX_LOG2_OUTPUTS:
        raise ValueError("log2_outputs must be 0, 1 or 2")
    if out not in ('int', 'bool'):
        raise ValueError("out must be 'int' or 'bool'")
    K, M, N = 1 << L, 1 << bits, 1024
    tables = numpy.asarray(tables)
    if L == 0:
        tables = tables[..., None, :]
    if tables.ndim < 2 or tables.shape[-2:] != (K, M):
        raise ValueError("tables must have shape batch + %s, got %s" % ((M,) if L == 0 else (K, M), tables.shape))
    if out == 'int':
        enc = (tables.astype(numpy.int64) % M) << (31 - bits)
    else:
        enc = numpy.where(tables != 0, int(MU), -int(MU)).astype(numpy.int64)
    i = numpy.arange(N)
    j = i & (K - 1)                       # output stored at position i
    box = N >> bits
    m = ((i - j) + box // 2) // box       # message whose box holds the phase i - j; M = the top half-box
    wrap = m == M
    vals = enc[..., j, numpy.where(wrap, 0, m)]
    vals = numpy.where(wrap, -vals, vals)
    return (vals & 0xffffffff).astype(numpy.uint32).view(numpy.int32)


# Multi-bit keys (bootstrap.py: MultiBitBootstrapKey) carry three times the blind-rotation variance (DESIGN.md section
# 14): the (P, L, shift) they allow, which follows from lut_sigma(..., multi_bit=2) (tests check it), and the standard
# deviations measured by tools/multibit_noise.py with a multi-bit key, keyed as MEASURED_SIGMA, on an H100 80GB HBM3
# (700 W, 1980 MHz), 65 536 inputs each.  All lie 2 - 3 % below the estimates; lut_sigma takes the larger of the two.
ALLOWED_MULTI_BIT = {
    (1, 0, None), (1, 1, None), (1, 2, None), (1, 0, 0), (1, 1, 0), (1, 2, 0),
    (2, 0, None), (2, 1, None), (2, 0, 0),
}
MEASURED_SIGMA_MULTI_BIT = {
    (0, None): 0.00586, (0, 0): 0.00804, (0, 1): 0.01237,
    (1, None): 0.00698, (1, 0): 0.00882, (1, 1): 0.01290,
    (2, None): 0.01035, (2, 0): 0.01167, (2, 1): 0.01505,
}


def _sigma_estimate(in_out_params, tgsw_params, ks_decomp_length, ks_log2_base, log2_outputs, shift, multi_bit=1):
    """Analytic standard deviation of the rounded phase of a LUT input that is one LUT output (shift None) or
    x * 2^shift + y of two: weight * (blind rotation + key switch) + mod-switch rounding.  A multi-bit key's rotation
    has n / 2 steps of 3 external products, each times X^k - 1, which doubles its variance: 3 n products' worth."""
    tl = tgsw_params.tlwe_params
    n, N, k = in_out_params.size, tl.polynomial_degree, tl.mask_size
    half_digit = 2**tgsw_params.bs_log2_base / 2
    products = 3 * n if multi_bit == 2 else n
    blind_rotation = products * (k + 1) * tgsw_params.decomp_length * N * half_digit**2 / 3 * tl.min_noise**2
    base = 2**ks_log2_base
    keyswitch = k * N * ks_decomp_length * (base - 1) / base * in_out_params.min_noise**2
    modswitch = (n / 2 + 1) * (2**log2_outputs / (2 * N))**2 / 12
    weight = 1 if shift is None else 4**shift + 1
    return (weight * (blind_rotation + keyswitch) + modswitch)**0.5


def _sigma(in_out_params, tgsw_params, ks_decomp_length, ks_log2_base, log2_outputs, shift, multi_bit=1):
    est = _sigma_estimate(in_out_params, tgsw_params, ks_decomp_length, ks_log2_base, log2_outputs, shift, multi_bit)
    if tgsw_params.tlwe_params.mask_size == 1:
        measured = MEASURED_SIGMA_MULTI_BIT if multi_bit == 2 else MEASURED_SIGMA
        est = max(est, measured.get((log2_outputs, shift), 0.0))
    return est


def lut_sigma(params, log2_outputs, shift=None, multi_bit=1):
    """The standard deviation `check_noise` uses for a NuFHEParameters set (estimate, or the measured value if larger);
    multi_bit=2 for a multi-bit bootstrap key."""
    return _sigma(params.in_out_params, params.tgsw_params, params.ks_decomp_length, params.ks_log2_base,
                  log2_outputs, shift, multi_bit)


def bootstrap_variance(params, multi_bit=1):
    """Estimated phase variance of a bootstrap output after the key switch: blind rotation + key switch."""
    return _sigma_estimate(params.in_out_params, params.tgsw_params, params.ks_decomp_length, params.ks_log2_base,
                           0, None, multi_bit)**2 - (params.in_out_params.size / 2 + 1) / (2 * 1024)**2 / 12


def _check_config(bits, log2_outputs, shift):
    _check_bits(bits)
    if not 0 <= log2_outputs <= MAX_LOG2_OUTPUTS:
        raise ValueError("log2_outputs must be 0, 1 or 2")
    if shift is not None and not 0 <= shift < bits:
        raise ValueError("shift must lie in [0, %d) for %d-bit messages" % (bits, bits))


def _check_margin(sigma, bits, log2_outputs, shift):
    margin = 2.0**-(bits + 2) / sigma
    if margin < MARGIN_SIGMAS:
        raise ValueError("a LUT with %d-bit messages, %d outputs and %s has %.1f sigma of noise margin, below %d"
                         % (bits, 1 << log2_outputs, 'one input' if shift is None else 'inputs x * 2^%d + y' % shift,
                            margin, MARGIN_SIGMAS))


def check_noise(params, bits, log2_outputs, shift=None, multi_bit=1):
    """Raise ValueError unless inputs that are LUT outputs (one, or x * 2^shift + y of two) stay 7 sigma inside their
    boxes of half-width 2^-(bits + 2); multi_bit=2 for a multi-bit bootstrap key."""
    _check_config(bits, log2_outputs, shift)
    _check_margin(lut_sigma(params, log2_outputs, shift, multi_bit), bits, log2_outputs, shift)


class LookupTable:
    """A device-resident test vector.  `tables`: batch + (2^bits,) for one output, batch + (2^L, 2^bits) for 2^L
    outputs of one input; an empty batch shape means one table for every ciphertext, otherwise the batch shape must be
    the ciphertexts' shape.  log2_outputs=None: a 1-D table has one output, a 2-D one has as many as rows (2 or 4)."""

    def __init__(self, thr, tables, bits, log2_outputs=None, out='int'):
        tables = numpy.asarray(tables)
        if log2_outputs is None:
            if tables.ndim == 1:
                log2_outputs = 0
            elif tables.ndim == 2 and tables.shape[0] in (2, 4):
                log2_outputs = tables.shape[0].bit_length() - 1
            else:
                raise ValueError("give log2_outputs for tables of shape %s" % (tables.shape,))
        tv = make_test_vector(tables, bits, log2_outputs, out)
        self.bits = int(bits)
        self.log2_outputs = int(log2_outputs)
        self.out = out
        self.batch_shape = tuple(tv.shape[:-1])
        self.tv = thr.to_device(tv)

    @property
    def outputs(self):
        return 1 << self.log2_outputs


def _expand(x, shape):
    a, b = x.a, x.b
    if tuple(b.shape) != shape:
        while b.dim() < len(shape):
            a, b = a.unsqueeze(0), b.unsqueeze(0)
        a, b = a.expand(shape + (a.shape[-1],)), b.expand(shape)
    return (a.contiguous().reshape(-1, a.shape[-1]), b.contiguous().reshape(-1))


def _lut_steps(thr, bk, p1, p2, s1, tv, L, B, perf_params):
    """The multi-kernel path, composed from the reference's steps: mod-switch with message space 2N / 2^L times 2^L,
    test-vector rotation, trivial accumulator, blind rotation, then per output j a rotation by X^(2N - j) and the
    sample extraction.  Returns (B * 2^L, k * N) and (B * 2^L,) like Engine.bootstrap_lut_extract."""
    accum_params = bk.bk_params.tlwe_params
    n, N, k = bk.in_out_params.size, accum_params.polynomial_degree, accum_params.mask_size
    K = 1 << L
    dev = p1[1].device
    xa, xb = torch.empty((B, n), dtype=torch.int32, device=dev), torch.empty((B,), dtype=torch.int32, device=dev)
    thr.lwe_affine((xa, xb), p1, p2, 0, s1, 1)
    bara, barb = torch.empty_like(xa), torch.empty_like(xb)
    t32_to_phase(thr, barb, xb, (2 * N) >> L)
    t32_to_phase(thr, bara, xa, (2 * N) >> L)
    if L:
        thr.lwe_affine((bara, barb), (bara, barb), None, 0, K, 0)
    source = TorusPolynomialArray(tv.expand(B, N).contiguous())
    testvectbis = TorusPolynomialArray.empty(thr, N, (B,))
    shift_tp_inverted_power(thr, testvectbis, barb, source)
    acc = TLweSampleArray.empty(thr, accum_params, (B,))
    tlwe_noiseless_trivial(thr, acc, testvectbis)
    blind_rotate(thr, acc, bk, bara, n, bk.bk_params, perf_params)
    out_a = torch.empty((B, K, k * N), dtype=torch.int32, device=dev)
    out_b = torch.empty((B, K), dtype=torch.int32, device=dev)
    ext = LweSampleArray.empty(thr, bk.extract_params, (B,))
    rotated = TLweSampleArray.empty(thr, accum_params, (B,))
    for j in range(K):
        src = acc
        if j:
            powers = torch.full((B,), 2 * N - j, dtype=torch.int32, device=dev)
            thr.shift_torus_polynomial(rotated.a.coeffs, acc.a.coeffs, powers, polys_per_power=k + 1,
                                       mode=thr.SHIFT_PLAIN)
            src = rotated
        tlwe_extract_lwe_samples(thr, ext, src)
        out_a[:, j].copy_(ext.a)
        out_b[:, j].copy_(ext.b)
    return out_a.reshape(B * K, k * N), out_b.reshape(B * K)


def bootstrap_lut(thr, results, bk, ks, table: LookupTable, x: LweSampleArray, y: LweSampleArray = None, shift=0,
                  perf_params=None):
    """results[j] = LWE(f_j(m)) with m the message of x, or of x * 2^shift + y when y is given.  `results` is a list of
    table.outputs ciphertexts (or one ciphertext for a one-output table), all of the same shape, to which x and y
    broadcast.  One fused launch when the key allows it (Engine.bootstrap_lut_extract), else the reference's separate
    steps; then one key switch of all 2^L samples.  Raises ValueError when the noise margin is too small."""
    if isinstance(results, LweSampleArray):
        results = [results]
    L = table.log2_outputs
    if len(results) != table.outputs:
        raise ValueError("a table with %d outputs needs %d results, got %d" % (table.outputs, table.outputs, len(results)))
    shape = tuple(results[0].shape)
    for r in results:
        if tuple(r.shape) != shape:
            raise ValueError("all results must have one shape")
    check_shape(results[0], *([x] if y is None else [x, y]))
    if table.batch_shape and table.batch_shape != shape:
        raise ValueError("per-ciphertext tables of shape %s do not match results of shape %s" % (table.batch_shape, shape))
    _check_config(table.bits, L, None if y is None else shift)
    _check_margin(_sigma(bk.in_out_params, bk.bk_params, ks.decomp_length, ks.log2_base, L,
                         None if y is None else shift, getattr(bk, 'multi_bit', 1)), table.bits, L,
                  None if y is None else shift)
    p1 = _expand(x, shape)
    p2 = _expand(y, shape) if y is not None else None
    s1 = 1 << shift if y is not None else 1
    tv = table.tv.reshape(-1, 1024) if table.batch_shape else table.tv
    keys = OneKey(thr, bk, ks, perf_params)
    ea, eb = keys.bootstrap_lut_extract(p1, p2, s1, tv, L)
    ra, rb, rcv = keys.keyswitch((ea, eb), want_cv=True)
    K = table.outputs
    ra, rb, rcv = ra.reshape(shape + (K, ra.shape[-1])), rb.reshape(shape + (K,)), rcv.reshape(shape + (K,))
    for j, r in enumerate(results):
        r.a.copy_(ra[..., j, :])
        r.b.copy_(rb[..., j])
        r.current_variances.copy_(rcv[..., j])
    return results
