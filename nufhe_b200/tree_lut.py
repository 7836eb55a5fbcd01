"""Tree-based programmable bootstrapping with encrypted test vectors (DESIGN.md section 13): lookup tables on several
encrypted digits of P = 1 or 2 bits each, with the parameters that `lut.ALLOWED` already accepts.

A table f of D digits d_{D-1} .. d_0 is evaluated one digit at a time.  Level 1 evaluates, for every value v of the
higher digits, the column f(v, d_0) with ordinary LUTs on d_0 (several columns per bootstrap, as many as the noise rule
allows).  Every following level takes the 2^P outputs that differ in its digit only, key-switches them into one GLWE
test vector under the bootstrap key's own GLWE key S (the tree key: GLWE_S encryptions of s_i g_j, seeded like the
packing key, ChaCha20 stream (seed, nonce 5)), and blind-rotates that encrypted test vector by its digit.  Every
bootstrap therefore takes a fresh LUT output as input; the noise grows by one blind rotation and key switch per level.
"""
import numpy
import torch

from .lwe import LweSampleArray
from .tlwe import TLweSampleArray, tlwe_extract_lwe_samples
from .numeric_functions import t32_to_phase
from .bootstrap import blind_rotate
from .gates import check_shape
from .packing import _GadgetKey, PACK_LEVELS, PACK_LOG2_BASE
from .batch_keys import OneKey
from . import lut

NONCE_TREE_KEY = 5
_TREE_KEY_TAG = 'nufhe_b200.NuFHETreeKey/1'
MAX_DIGITS = 8                      # an upper bound on D whatever the noise allows (a table has 2^(P D) entries)
ROWS_PER_PASS = 1 << 16             # level-1 bootstraps per pass: bounds the device memory whatever the batch

# Standard deviations (torus units) of the rounded mod-switched phase of a level-D tree output used as a one-input LUT
# input, measured by tools/tree_lut_noise.py for the default parameter set over 65 536 outputs per entry, keyed by
# (P, D), on an H100 80GB HBM3 (700 W, 1980 MHz) (DESIGN.md section 13).  All lie within 0.5 % of the estimates;
# tree_sigma takes the larger of the two.
MEASURED_SIGMA = {
    (2, 2): 0.00619, (2, 3): 0.00743, (2, 4): 0.00846,
    (1, 2): 0.00622, (1, 3): 0.00742, (1, 4): 0.00849,
}
# The same with a multi-bit bootstrap key (tools/multibit_noise.py, same card and count; DESIGN.md section 14), up to
# one level past what the rule allows.  All lie 2 - 3 % below the estimates.
MEASURED_SIGMA_MULTI_BIT = {
    (2, 2): 0.00804, (2, 3): 0.00971,
    (1, 2): 0.00803, (1, 3): 0.00974, (1, 4): 0.01116,
}


class NuFHETreeKey(_GadgetKey):
    """The key of tree-based LUTs: params, the seed of the masks, the bodies (n, t, N) int32 (4.1 MB for k = 1) and
    the variance of their noise.  Row i t + j is a GLWE encryption under the bootstrap key's GLWE key S of the constant
    s_i g_j.  Made with the cloud key (`ctx.make_cloud_key(sk, tree_key=True)`), since S exists only during that call.
    `planes(thr)` -- the byte planes nb_tree_keyswitch reads, 8.4 MB for k = 1 -- is built once per engine and cached."""
    NONCE = NONCE_TREE_KEY
    TAG = _TREE_KEY_TAG
    NAME = 'tree key'

    def __init__(self, params, seed, body, variance: float):
        super().__init__(params, seed, body, variance)
        self._planes = None

    @classmethod
    def from_secret_key(cls, thr, rng, secret_key, tgsw_key):
        """Draws the seed, then the Gaussian body noises (n, t, N) with tlwe_params.min_noise."""
        return cls._encrypt(thr, rng, secret_key, tgsw_key.tlwe_key.key.coeffs)

    def planes(self, thr):
        if self._planes is None or self._planes[0] is not thr:
            self._planes = (thr, thr.tree_prepare(self.masks(thr), self.body.to(thr.device)))
        return self._planes[1]


# ---------------------------------------------------------------- noise

def _modswitch_variance(params, log2_outputs=0):
    n, N = params.in_out_params.size, params.tgsw_params.tlwe_params.polynomial_degree
    return (n / 2 + 1) * (2**log2_outputs / (2 * N))**2 / 12


def level_variance(params, multi_bit=1):
    """Blind rotation + key switch of one level: the estimate of lut._sigma_estimate, or for k = 1 the measured
    one-output LUT variance less its mod-switch term when that is larger (multi_bit=2: a multi-bit bootstrap key)."""
    est = lut._sigma_estimate(params.in_out_params, params.tgsw_params, params.ks_decomp_length, params.ks_log2_base,
                              0, None, multi_bit)**2 - _modswitch_variance(params)
    measured = (lut.MEASURED_SIGMA_MULTI_BIT if multi_bit == 2 else lut.MEASURED_SIGMA).get((0, None))
    if params.tgsw_params.tlwe_params.mask_size == 1 and measured:
        est = max(est, measured**2 - _modswitch_variance(params))
    return est


def test_vector_variance(params, bits):
    """What an encrypted test vector adds per level: the box sum of the key noise, box n t E[d^2] sigma^2, and the
    rounding of the masks to 16 bits, (n / 2) 2^-32 / 12."""
    tl = params.tgsw_params.tlwe_params
    n, N = params.in_out_params.size, tl.polynomial_degree
    base = 2**PACK_LOG2_BASE
    e_d2 = (base**2 - 1) / 12 + 0.25            # digits uniform in [-128, 127]
    key = (N >> bits) * n * PACK_LEVELS * e_d2 * tl.min_noise**2
    rounding = n / 2 * 2.0**-32 / 12
    return key + rounding


def output_variance(params, bits, digits, multi_bit=1):
    """Phase variance of a level-`digits` output: D levels of blind rotation and key switch, D - 1 encrypted test
    vectors."""
    return digits * level_variance(params, multi_bit) + (digits - 1) * test_vector_variance(params, bits)


def tree_sigma(params, bits, digits, multi_bit=1):
    """Standard deviation of the rounded phase of a level-`digits` tree output used as a one-input LUT input: the
    output variance plus the mod-switch; the measured value if larger."""
    sigma = (output_variance(params, bits, digits, multi_bit) + _modswitch_variance(params))**0.5
    if params.tgsw_params.tlwe_params.mask_size == 1:
        measured = MEASURED_SIGMA_MULTI_BIT if multi_bit == 2 else MEASURED_SIGMA
        sigma = max(sigma, measured.get((bits, digits), 0.0))
    return sigma


def max_digits(params, bits, multi_bit=1):
    """The largest D whose outputs stay lut.MARGIN_SIGMAS standard deviations inside their boxes (4 for P = 2; 2 with
    a multi-bit bootstrap key)."""
    best = 0
    for d in range(1, MAX_DIGITS + 1):
        if 2.0**-(bits + 2) / tree_sigma(params, bits, d, multi_bit) >= lut.MARGIN_SIGMAS:
            best = d
    return best


def _check_config(params, bits, digits, multi_bit=1):
    if bits not in (1, 2):
        raise ValueError('tree LUTs take digits of 1 or 2 bits, got %r' % (bits,))
    top = max_digits(params, bits, multi_bit)
    if int(digits) != digits or not 2 <= digits <= top:
        raise ValueError('a tree LUT on %d-bit digits takes 2 to %d digits with these parameters, got %r'
                         % (bits, top, digits))


def _level1_log2_outputs(params, bits, columns, multi_bit=1):
    """Columns per level-1 bootstrap: the largest 2^L (L <= 2, 2^L <= columns) that the LUT noise rule allows."""
    best = 0
    for L in range(lut.MAX_LOG2_OUTPUTS + 1):
        if (1 << L) <= columns and 2.0**-(bits + 2) / lut.lut_sigma(params, L, None, multi_bit) >= lut.MARGIN_SIGMAS:
            best = L
    return best


# ---------------------------------------------------------------- tables and evaluation

class TreeLookupTable:
    """F functions of D digits of `bits` bits: tables of shape (F,) + (2^bits,) * D, or (2^bits,) * D for F = 1, indexed
    [f, d_{D-1}, ..., d_0].  Holds the device-resident level-1 test vectors: the F 2^(bits (D-1)) columns f(v, .) in
    groups of 2^L (zero columns pad the last group), `tv` (Q, N) for Q = ceil(columns / 2^L)."""

    def __init__(self, thr, params, tables, bits, digits, out='int', multi_bit=1):
        """multi_bit=2: a table for a VM whose cloud key has a multi-bit bootstrap key (its noise rules)."""
        _check_config(params, bits, digits, multi_bit)
        self.multi_bit = multi_bit
        if out not in ('int', 'bool'):
            raise ValueError("out must be 'int' or 'bool'")
        M = 1 << bits
        tables = numpy.asarray(tables)
        self.single = tables.shape == (M,) * digits
        if self.single:
            tables = tables[None]
        if tables.ndim != digits + 1 or tables.shape[1:] != (M,) * digits:
            raise ValueError('tables of %d functions of %d %d-bit digits have shape (F,) + %s, got %s'
                             % (tables.shape[0] if tables.ndim else 0, digits, bits, (M,) * digits, tables.shape))
        self.params = params
        self.bits, self.digits, self.out = int(bits), int(digits), out
        self.functions = tables.shape[0]
        self.columns = self.functions * M**(digits - 1)
        self.log2_outputs = _level1_log2_outputs(params, bits, self.columns, multi_bit)
        K = 1 << self.log2_outputs
        self.groups = -(-self.columns // K)
        cols = numpy.zeros((self.groups * K, M), numpy.int64)
        cols[:self.columns] = tables.reshape(self.columns, M)
        grouped = cols.reshape(self.groups, K, M) if K > 1 else cols
        self.tv = thr.to_device(lut.make_test_vector(grouped, bits, self.log2_outputs, out))

    def reserve_batch(self, batch):
        """The `reserve_batch` a `vm.capture` of lut_tree on `batch` ciphertexts needs: the level-1 key switch of one
        pass."""
        per = self.groups << self.log2_outputs
        return min(batch, max(1, ROWS_PER_PASS // self.groups)) * per


def _level1(keys, table, d0):
    """(B, n) masks and (B,) bodies of one digit -> LWE (B, columns) of f(v, d_0) for every column v."""
    a, b = d0
    B, n = a.shape
    Q, L = table.groups, table.log2_outputs
    K = 1 << L
    ea_ = a[:, None, :].expand(B, Q, n).reshape(B * Q, n)
    eb_ = b[:, None].expand(B, Q).reshape(B * Q)
    tv = table.tv.reshape(Q, -1)[None].expand(B, Q, table.tv.shape[-1]).reshape(B * Q, -1)
    ea, eb = keys.bootstrap_lut_extract((ea_, eb_), None, 1, tv, L, per=Q)
    ra, rb, _ = keys.keyswitch((ea, eb), per=Q * K)
    return ra.reshape(B, Q * K, n)[:, :table.columns], rb.reshape(B, Q * K)[:, :table.columns]


def _glwe_steps(thr, bk, x, tv, perf_params):
    """The encrypted-test-vector bootstrap as separate steps (any k): mod-switch, X^(2N - barb) on all k+1
    polynomials of tv, blind rotation of that accumulator, extraction.  Returns a (T, k N), b (T,)."""
    accum_params = bk.bk_params.tlwe_params
    N, n = accum_params.polynomial_degree, bk.in_out_params.size
    xa, xb = x
    T = xb.shape[0]
    bara, barb = torch.empty_like(xa), torch.empty_like(xb)
    t32_to_phase(thr, barb, xb, 2 * N)
    t32_to_phase(thr, bara, xa, 2 * N)
    acc = TLweSampleArray.empty(thr, accum_params, (T,))
    thr.shift_torus_polynomial(acc.a.coeffs, tv, barb, polys_per_power=accum_params.mask_size + 1,
                               mode=thr.SHIFT_INVERT)
    blind_rotate(thr, acc, bk, bara, n, bk.bk_params, perf_params)
    ext = LweSampleArray.empty(thr, bk.extract_params, (T,))
    tlwe_extract_lwe_samples(thr, ext, acc)
    return ext.a, ext.b


def _level(keys, table, cur, digit):
    """One level >= 2: cur (B, W, n) / (B, W) LWE outputs whose last 2^bits entries differ in this level's digit ->
    (B, W / 2^bits, n) / (B, W / 2^bits)."""
    ca, cb = cur
    B, W, n = ca.shape
    M = 1 << table.bits
    k = table.params.tgsw_params.tlwe_params.mask_size
    T = B * (W // M)
    v = keys.tree_keyswitch(ca.reshape(B * W, n), k, per=W)
    tv = keys.thr.tree_assemble(v.reshape(T, M, k + 1, -1), cb.reshape(T, M), table.bits)
    da, db = digit
    xa = da[:, None, :].expand(B, W // M, n).reshape(T, n)
    xb = db[:, None].expand(B, W // M).reshape(T)
    ea, eb = keys.bootstrap_glwe_lut_extract((xa, xb), tv, per=W // M)
    ra, rb, _ = keys.keyswitch((ea, eb), per=W // M)
    return ra.reshape(B, W // M, n), rb.reshape(B, W // M)


def evaluate(keys, table, flat):
    """The tree LUT on the batch `flat` (the D digits as (a (B, n), b (B,)), d_0 first) with `keys` (batch_keys):
    out_a (B, F, n) and out_b (B, F), at most ROWS_PER_PASS level-1 bootstraps per pass."""
    thr = keys.thr
    B, n = flat[0][0].shape
    out_a, out_b = thr.empty((B, table.functions, n), torch.int32), thr.empty((B, table.functions), torch.int32)
    step = max(1, ROWS_PER_PASS // table.groups)
    for c0 in range(0, B, step):
        c1 = min(B, c0 + step)
        part = [(a[c0:c1], b[c0:c1]) for a, b in flat]
        pass_keys = keys.split(c0, c1)
        cur = _level1(pass_keys, table, part[0])
        for level in range(1, table.digits):
            cur = _level(pass_keys, table, cur, part[level])
        out_a[c0:c1].copy_(cur[0])
        out_b[c0:c1].copy_(cur[1])
    return out_a, out_b


def lut_tree(thr, results, bk, ks, tree_key, table: TreeLookupTable, digits, perf_params=None):
    """results[f] = LWE(f(d_{D-1}, ..., d_0)) for the digit ciphertexts `digits` = [d_{D-1}, ..., d_0] (one shape, or
    shapes that broadcast to the results' shape).  Raises TypeError unless tree_key is a NuFHETreeKey, ValueError for a
    wrong digit count, mismatched shapes or parameters."""
    if not isinstance(tree_key, NuFHETreeKey):
        raise TypeError('lut_tree needs a NuFHETreeKey (ctx.make_cloud_key(sk, tree_key=True)), got %s'
                        % type(tree_key).__name__)
    if not isinstance(table, TreeLookupTable):
        raise TypeError('lut_tree needs a TreeLookupTable (vm.make_tree_lut), got %s' % type(table).__name__)
    if tree_key.params != table.params:
        raise ValueError('the tree key was made for other parameters than this table')
    if getattr(bk, 'multi_bit', 1) != table.multi_bit:
        raise ValueError('the table was made for another kind of bootstrap key (multi_bit=%d, the key has %d): make it '
                         'with this VM' % (table.multi_bit, getattr(bk, 'multi_bit', 1)))
    digits = list(digits)
    if len(digits) != table.digits:
        raise ValueError('the table takes %d digits, got %d' % (table.digits, len(digits)))
    if len(results) != table.functions:
        raise ValueError('the table has %d functions, got %d results' % (table.functions, len(results)))
    shape = tuple(results[0].shape)
    for r in results:
        if tuple(r.shape) != shape:
            raise ValueError('all results must have one shape')
    check_shape(results[0], *digits)
    for d in digits:
        if tuple(d.shape) != tuple(digits[0].shape):
            raise ValueError('all digits must have one shape, got %s and %s' % (tuple(digits[0].shape), tuple(d.shape)))
    flat = [lut._expand(d, shape) for d in reversed(digits)]    # d_0 first
    out_a, out_b = evaluate(OneKey(thr, bk, ks, perf_params, tree_key=tree_key), table, flat)
    out_a, out_b = out_a.reshape(shape + out_a.shape[1:]), out_b.reshape(shape + out_b.shape[1:])
    for f, r in enumerate(results):
        r.a.copy_(out_a[..., f, :])
        r.b.copy_(out_b[..., f])
        r.current_variances.fill_(float(output_variance(table.params, table.bits, table.digits)))
    return results
