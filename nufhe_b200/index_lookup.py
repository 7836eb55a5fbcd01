"""Encrypted-index table lookups (DESIGN.md section 15): the client encrypts every bit of an index as a TGSW sample
(a selector) under the bootstrap key's GLWE key S; the server looks the index up in a plaintext table with CMux gates
alone and returns ordinary LWE ciphertexts under the user's key.  No bootstrap is involved.

An index 0 <= idx < 2^m (1 <= m <= 20) is m selectors C_j = Z_j + b_j H, b_j = (idx >> j) & 1.  A table of W columns of
2^m entries is laid out in GLWE plaintext polynomials:
  * m >= 10: column w is 2^(m-10) polynomials, entry i at coefficient i mod 1024 of polynomial i >> 10;
  * m < 10: one polynomial for all columns, entry (w, i) at coefficient i + w 2^m (W 2^m <= 1024).
Evaluation: a CMux tree over the polynomials for the bits j = 10 .. m-1 (d_2i + C_j [x] (d_2i+1 - d_2i), the first
level reading the table as trivial samples (0, T)), then for j < min(m, 10) the blind-rotation step with the constant
rotation 2N - 2^j, ACC <- ACC + C_j [x] ((X^(-2^j) - 1) ACC), which leaves X^(-idx mod 1024) ACC; sample extraction at
coefficient w 2^m (m < 10) or 0 (m >= 10) and the cloud key's key switch (S -> s).

Each external product runs the exact FP64 step of the bootstrap (nb_index_cmux_level, nb_index_rotate_extract) on the
selector spectra (nb_index_prepare); results equal an exact-integer computation bit for bit.  Unlike the bootstrap, the
gadget decomposition rounds to the nearest multiple of 2^12 instead of truncating, so that its error is centred and
does not shift the phase coherently along the m CMuxes (DESIGN.md section 15).
"""
import io
import pickle

import numpy
import torch

from .lwe import LweSampleArray
from .tlwe import TLweKey, TLweSampleArray, tlwe_encrypt_zero, tlwe_encrypt_zero_with_masks
from .tgsw import TGswKey, TGswSampleArray, tgsw_encrypt_int
from .polynomials import IntPolynomialArray
from .compressed import draw_seed, _check_tag, _variance, _wrap32, tgsw_add_message_seeded
from .random_numbers import rand_gaussian_torus32
from .gates import MU
from .batch_keys import owners
from . import compact, lut, packing

NONCE_INDEX = 6
MAX_BITS = 20
N = 1024
ROTATE_BITS = 10                        # log2 N: the low bits are taken by the rotation, the others by the tree
NODE_BYTES = 2 * N * 4                  # one GLWE sample (k = 1)
# Device scratch of one pass of vm.lookup: the FP64 spectra of the selectors (128 KB per bit and query) and the CMux-tree
# nodes (8 KB each, W 2^(m-10) per query at most: 4 MB at m = 20, W = 1).  A batch is cut into as many passes as that
# takes (queries_per_pass), whatever its size.
PASS_BYTES = 2 << 30

_SECRET_KEY_TAG = 'nufhe_b200.NuFHEIndexSecretKey/1'
_INDEX_TAG = 'nufhe_b200.EncryptedIndexArray/1'
_COMPRESSED_INDEX_TAG = 'nufhe_b200.CompressedEncryptedIndexArray/1'
_ENCRYPTED_TABLE_TAG = 'nufhe_b200.EncryptedIndexTable/1'


def _check_params(params):
    tl = params.tgsw_params.tlwe_params
    if tl.mask_size != 1:
        raise ValueError('encrypted-index lookups run on the FP64 CMux step, which takes tlwe_mask_size = 1 only, got %d'
                         % tl.mask_size)
    tg = params.tgsw_params
    if tg.decomp_length != 2 or tg.bs_log2_base != 10 or tl.polynomial_degree != N:
        raise ValueError('encrypted-index lookups take N = 1024, l = 2, Bg = 2^10')


def _check_bits(bits):
    if isinstance(bits, bool) or int(bits) != bits or not 1 <= bits <= MAX_BITS:
        raise ValueError('an encrypted index has 1 to %d bits, got %r' % (MAX_BITS, bits))
    return int(bits)


# ---------------------------------------------------------------- noise

def cmux_variance(params):
    """What one external product with a fresh selector adds through the selector's noise:
    (k+1) l N ((Bg/2)^2 / 3) bs_stdev^2 (1.84e-8)."""
    tg = params.tgsw_params
    tl = tg.tlwe_params
    return (tl.mask_size + 1) * tg.decomp_length * tl.polynomial_degree * (2**tg.bs_log2_base / 2)**2 / 3 * tl.min_noise**2


def decomposition_variance(params):
    """What one external product adds through the gadget decomposition when the selector bit is 1: the rounded digits
    (index_lookup.cuh) leave an error uniform over a step of 2^-(l log2 Bg) on every coefficient, on the body and,
    through the key, on about k N / 2 mask coefficients: (1 + k N / 2) 2^(-2 l log2 Bg) / 12 (3.9e-11).  Centred, so
    it does not accumulate along the m CMuxes beyond this variance."""
    tg = params.tgsw_params
    tl = tg.tlwe_params
    return (1 + tl.mask_size * tl.polynomial_degree / 2) * 2.0**(-2 * tg.decomp_length * tg.bs_log2_base) / 12


def keyswitch_variance(params):
    """The key switch: k N t (base-1)/base ks_stdev^2 (3.6e-6, DESIGN.md section 9)."""
    tl = params.tgsw_params.tlwe_params
    base = 2**params.ks_log2_base
    return tl.mask_size * tl.polynomial_degree * params.ks_decomp_length * (base - 1) / base * params.in_out_params.min_noise**2


def extracted_variance(params, m):
    """Variance of a lookup result before the key switch: one CMux per index bit (tree levels and rotation steps)."""
    return m * (cmux_variance(params) + decomposition_variance(params))


def output_variance(params, m):
    return extracted_variance(params, m) + keyswitch_variance(params)


def rounding_variance(params):
    """The 16-bit rounding of a stored GLWE leaf: the k N mask coefficients, each multiplied by a key bit, and the body,
    (k N / 2 + 1) 2^-32 / 12 (9.9e-9)."""
    tl = params.tgsw_params.tlwe_params
    return (tl.mask_size * tl.polynomial_degree / 2 + 1) * 2.0**-32 / 12


def packing_variance(params):
    """What packing LWE samples into a leaf adds (DESIGN.md section 12, with the tree key in place of the packing key):
    the key noise n t N E[d^2] sigma^2, the 16-bit rounding of the input masks (n / 2) 2^-32 / 12 and the rounding of
    the leaf (3.03e-7)."""
    tl = params.tgsw_params.tlwe_params
    n = params.in_out_params.size
    e_d2 = (2**(2 * packing.PACK_LOG2_BASE) - 1) / 12 + 0.25        # digits uniform in [-128, 127]
    key = n * packing.PACK_LEVELS * tl.polynomial_degree * e_d2 * tl.min_noise**2
    return key + n / 2 * 2.0**-32 / 12 + rounding_variance(params)


def write_variance(params, m, lwe_values=True):
    """What one query of a write adds to every entry of the table (DESIGN.md section 21): the m external products of its
    rotation and demultiplexer, extracted_variance(m), and with LWE values the tree key's noise on every coefficient of
    the delta, n t E[d^2] sigma^2 (the key term of test_vector_variance without the box sum)."""
    tl = params.tgsw_params.tlwe_params
    e_d2 = (2**(2 * packing.PACK_LOG2_BASE) - 1) / 12 + 0.25
    key = params.in_out_params.size * packing.PACK_LEVELS * e_d2 * tl.min_noise**2 if lwe_values else 0.0
    return extracted_variance(params, m) + key


def value_variance(params, variance):
    """What an LWE value of `variance` brings to the entry it is written to: its own noise and the truncation of its
    mask to the tree key's 16 bits, (n / 2) 2^-32 / 12."""
    return variance + params.in_out_params.size / 2 * 2.0**-32 / 12


def table_sigma(params, leaf_variance, m, out):
    """Standard deviation of the rounded phase of what a lookup result of the table feeds: a one-input vm.lut for an
    'int' table, a two-input gate (the weight of lut's x + y inputs) for a 'bool' table."""
    return lut_input_sigma(params, leaf_variance, m) if out == 'int' else lut_input_sigma(params, leaf_variance, m, 0, 0)


def _box(out, bits_out):
    return 2.0**-((bits_out if out == 'int' else 1) + 2)


def check_table_variance(params, leaf_variance, m, out, bits_out):
    """ValueError unless lookups into a table whose leaves carry `leaf_variance` keep lut.MARGIN_SIGMAS."""
    margin = _box(out, bits_out) / table_sigma(params, leaf_variance, m, out)
    if margin < lut.MARGIN_SIGMAS:
        raise ValueError('the written table would keep %.1f sigma of noise margin on its lookups, below %d: '
                         'refresh_table it first' % (margin, lut.MARGIN_SIGMAS))


def max_table_variance(params, m, out, bits_out):
    """The largest leaf variance check_table_variance accepts (negative when even a noiseless table falls short)."""
    shift = None if out == 'int' else 0
    weight = 1 if shift is None else 2
    extra = ((_box(out, bits_out) / lut.MARGIN_SIGMAS)**2 - lut.lut_sigma(params, 0, shift)**2) / weight
    return extra + lut.bootstrap_variance(params) - output_variance(params, m)


def written_table_variance(params, leaf_variance, m, queries, value_variances=None, write=False):
    """The leaf variance of a table after one call of `queries` queries: every entry gains queries * write_variance and
    the 16-bit rounding.  scatter_add of LWE values (value_variances, one per query) adds them all, as repeated indexes
    add up; `write` replaces its entries by values that carry their own noise and the lookup's, not the old leaf's."""
    lwe = value_variances is not None
    common = queries * write_variance(params, m, lwe) + rounding_variance(params)
    if not lwe:
        return leaf_variance + common
    vv = [value_variance(params, v) for v in value_variances]
    if write:
        return max(leaf_variance, max(vv, default=0.0) + output_variance(params, m)) + common
    return leaf_variance + sum(vv) + common


def writes_before_refresh(params, m, out, bits_out, lwe_values=False):
    """How many one-query calls a refreshed table (leaves of a bootstrap output plus packing_variance) takes before the
    next would be refused: scatter_adds of plain counts, or (lwe_values) writes of bootstrap outputs."""
    limit = max_table_variance(params, m, out, bits_out)
    v = lut.bootstrap_variance(params) + packing_variance(params)
    count = 0
    while True:
        v = written_table_variance(params, v, m, 1, [lut.bootstrap_variance(params)] if lwe_values else None, lwe_values)
        if v > limit:
            return count
        count += 1


def lut_input_sigma(params, leaf_variance, m, log2_outputs=0, shift=None):
    """Standard deviation of the rounded phase of a vm.lut input made of results of an m-bit lookup whose leaves carry
    `leaf_variance`: lut.lut_sigma (measured where larger) plus whatever such a result carries beyond a LUT output,
    weighted as the LUT weights its inputs.  For packed leaves (a LUT or gate output plus packing_variance) every
    configuration of lut.ALLOWED keeps lut.MARGIN_SIGMAS (DESIGN.md section 20)."""
    extra = max(0.0, leaf_variance + output_variance(params, m) - lut.bootstrap_variance(params))
    weight = 1 if shift is None else 4**shift + 1
    return (lut.lut_sigma(params, log2_outputs, shift)**2 + weight * extra)**0.5


def output_sigma(params, m):
    """Standard deviation (torus units) of a lookup result on m index bits: 2.0e-3 at m = 20 (variance 4.0e-6), below
    a gate output's 1.28e-5."""
    return output_variance(params, m)**0.5


# ---------------------------------------------------------------- keys and client-side arrays

class NuFHEIndexSecretKey:
    """The client's key for encrypted indices: params and the GLWE key S (k, N) int32 of the cloud key's bootstrap key.
    Made with the cloud key (`ctx.make_cloud_key(sk, index_key=True)`), since S exists only during that call; kept
    next to the NuFHESecretKey, which decrypts the lookup results."""

    def __init__(self, params, key):
        _check_params(params)
        self.params = params
        self.key = key
        if tuple(key.shape) != (1, N):
            raise ValueError('an index secret key has shape %s, got %s' % ((1, N), tuple(key.shape)))

    @classmethod
    def from_tgsw_key(cls, params, tgsw_key):
        """Draws nothing: S is the TLWE key of the TGSW key."""
        return cls(params, tgsw_key.tlwe_key.key.coeffs)

    def _tgsw_key(self):
        tl = self.params.tgsw_params.tlwe_params
        return TGswKey(self.params.tgsw_params, TLweKey(tl, IntPolynomialArray(self.key)))

    def dump(self, file_obj):
        pickle.dump(_SECRET_KEY_TAG, file_obj)
        pickle.dump(self.params, file_obj)
        pickle.dump(self.key.cpu().numpy(), file_obj)

    def dumps(self):
        file_obj = io.BytesIO()
        self.dump(file_obj)
        return file_obj.getvalue()

    @classmethod
    def load(cls, file_obj, thr):
        _check_tag(file_obj, _SECRET_KEY_TAG)
        params = pickle.load(file_obj)
        return cls(params, thr.to_device(pickle.load(file_obj)))

    @classmethod
    def loads(cls, s: bytes, thr):
        return cls.load(io.BytesIO(s), thr)

    def __eq__(self, other):
        return (self.__class__ == other.__class__ and self.params == other.params
                and torch.equal(self.key.cpu(), other.key.cpu()))


class EncryptedIndexArray:
    """Encrypted indices: params, the bit count m and the selectors `samples`, shape + (m, 2, 2, 2, N) int32 (TGSW
    samples under S, 32 KB per bit), and the variance of their noise."""

    def __init__(self, params, bits, samples, variance: float):
        _check_params(params)
        self.params = params
        self.bits = _check_bits(bits)
        self.samples = samples
        self.variance = float(variance)
        if samples.dim() < 5 or tuple(samples.shape[-5:]) != (self.bits, 2, 2, 2, N) or samples.dtype != torch.int32:
            raise ValueError('selectors of %d-bit indices are int32 shape + %s, got %s %s'
                             % (self.bits, (self.bits, 2, 2, 2, N), samples.dtype, tuple(samples.shape)))
        self.shape = tuple(samples.shape[:-5])

    def dump(self, file_obj):
        pickle.dump(_INDEX_TAG, file_obj)
        pickle.dump(self.params, file_obj)
        pickle.dump(self.bits, file_obj)
        pickle.dump(self.samples.cpu().numpy(), file_obj)
        pickle.dump(self.variance, file_obj)

    def dumps(self):
        file_obj = io.BytesIO()
        self.dump(file_obj)
        return file_obj.getvalue()

    @classmethod
    def _load_body(cls, file_obj, thr):
        params = pickle.load(file_obj)
        bits = pickle.load(file_obj)
        samples = thr.to_device(pickle.load(file_obj))
        return cls(params, bits, samples, pickle.load(file_obj))

    @classmethod
    def load(cls, file_obj, thr):
        _check_tag(file_obj, _INDEX_TAG)
        return cls._load_body(file_obj, thr)

    @classmethod
    def loads(cls, s: bytes, thr):
        return cls.load(io.BytesIO(s), thr)

    def __eq__(self, other):
        return (self.__class__ == other.__class__ and self.params == other.params and self.bits == other.bits
                and torch.equal(self.samples.cpu(), other.samples.cpu()) and self.variance == other.variance)


def _index_masks(thr, seed, rows):
    """The TLWE masks (rows, k+1, l, k, N) of `rows` selector rows: the ChaCha20 stream (seed, NONCE_INDEX)."""
    return thr.seeded_uniform(seed, NONCE_INDEX, (rows, 2, 2, 1, N))


class CompressedEncryptedIndexArray:
    """Encrypted indices without their masks: params, shape, bit count, the 256-bit seed of the masks and the bodies,
    shape + (m, 2, 2, N) int32 (16 KB per bit).  Rows for the mask polynomial carry the phase-equivalent body of
    compressed.tgsw_add_message_seeded.  `decompress(thr)` gives the EncryptedIndexArray that vm.lookup takes."""

    def __init__(self, params, shape, bits, seed, body, variance: float):
        _check_params(params)
        self.params = params
        self.shape = tuple(int(s) for s in shape)
        self.bits = _check_bits(bits)
        self.seed = numpy.asarray(seed, numpy.uint32).reshape(8)
        self.body = body
        self.variance = float(variance)
        if tuple(body.shape) != self.shape + (self.bits, 2, 2, N):
            raise ValueError('bodies of shape %s do not match %s' % (tuple(body.shape), self.shape + (self.bits, 2, 2, N)))

    def decompress(self, thr):
        rows = int(numpy.prod(self.shape, dtype=numpy.int64)) * self.bits
        samples = thr.empty((rows, 2, 2, 2, N), torch.int32)
        samples[..., :1, :] = _index_masks(thr, self.seed, rows)
        samples[..., 1, :] = self.body.to(samples.device).reshape(rows, 2, 2, N)
        return EncryptedIndexArray(self.params, self.bits, samples.reshape(self.shape + (self.bits, 2, 2, 2, N)),
                                   self.variance)

    def dump(self, file_obj):
        pickle.dump(_COMPRESSED_INDEX_TAG, file_obj)
        pickle.dump(self.params, file_obj)
        pickle.dump(self.shape, file_obj)
        pickle.dump(self.bits, file_obj)
        pickle.dump(self.seed, file_obj)
        pickle.dump(self.body.cpu().numpy(), file_obj)
        pickle.dump(self.variance, file_obj)

    def dumps(self):
        file_obj = io.BytesIO()
        self.dump(file_obj)
        return file_obj.getvalue()

    @classmethod
    def _load_body(cls, file_obj, thr):
        params = pickle.load(file_obj)
        shape = pickle.load(file_obj)
        bits = pickle.load(file_obj)
        seed = pickle.load(file_obj)
        body = thr.to_device(pickle.load(file_obj))
        return cls(params, shape, bits, seed, body, pickle.load(file_obj))

    @classmethod
    def load(cls, file_obj, thr):
        _check_tag(file_obj, _COMPRESSED_INDEX_TAG)
        return cls._load_body(file_obj, thr)

    @classmethod
    def loads(cls, s: bytes, thr):
        return cls.load(io.BytesIO(s), thr)

    def __eq__(self, other):
        return (self.__class__ == other.__class__ and self.params == other.params and self.shape == other.shape
                and self.bits == other.bits and (self.seed == other.seed).all()
                and torch.equal(self.body.cpu(), other.body.cpu()) and self.variance == other.variance)


def load_encrypted_index(file_obj, thr):
    """An EncryptedIndexArray or a CompressedEncryptedIndexArray, whichever the pickle holds (ValueError otherwise)."""
    try:
        tag = pickle.load(file_obj)
    except Exception as e:
        raise ValueError('not an encrypted index pickle: %s' % e) from e
    if tag == _INDEX_TAG:
        return EncryptedIndexArray._load_body(file_obj, thr)
    if tag == _COMPRESSED_INDEX_TAG:
        return CompressedEncryptedIndexArray._load_body(file_obj, thr)
    raise ValueError('not an encrypted index pickle (format tag %r)' % (tag if isinstance(tag, str) else type(tag).__name__))


def index_bits(values, bits):
    """The bits (idx >> j) & 1 of every index, shape + (bits,) int32; ValueError for values outside [0, 2^bits)."""
    bits = _check_bits(bits)
    values = numpy.asarray(values)
    if values.dtype.kind not in 'iu' and values.size:
        raise ValueError('indices must be integers, got %s' % values.dtype)
    values = values.astype(numpy.int64)
    if values.size and (values.min() < 0 or values.max() >= 2**bits):
        raise ValueError('indices must lie in [0, %d)' % 2**bits)
    return ((values[..., None] >> numpy.arange(bits)) & 1).astype(numpy.int32)


def encrypt_index(thr, rng, key: NuFHEIndexSecretKey, values, bits, compressed=False):
    """Selectors of the indices `values` (any shape): TGSW encryptions under S of their bits with the bootstrap key's
    noise.  Draws the masks and noises as tgsw_encrypt_int, or with compressed=True the seed, then the body noises."""
    if not isinstance(key, NuFHEIndexSecretKey):
        raise TypeError('encrypt_index needs a NuFHEIndexSecretKey (ctx.make_cloud_key(sk, index_key=True)), got %s'
                        % type(key).__name__)
    msgs = index_bits(values, bits)
    bits = msgs.shape[-1]
    shape = msgs.shape[:-1]
    rows = msgs.size
    params = key.params
    tg = params.tgsw_params
    noise = tg.tlwe_params.min_noise
    tkey = key._tgsw_key()
    arr = TGswSampleArray.empty(thr, tg, (rows,))
    m = thr.to_device(msgs.reshape(-1))
    if not compressed:
        tgsw_encrypt_int(thr, rng, arr, m, noise, tkey)
        return EncryptedIndexArray(params, bits, arr.samples.a.coeffs.reshape(shape + (bits, 2, 2, 2, N)), _variance(noise))
    seed = draw_seed(rng)
    noises = rand_gaussian_torus32(thr, rng, 0, noise, (rows, 2, 2, N))
    tlwe_encrypt_zero_with_masks(thr, arr.samples, _index_masks(thr, seed, rows), noises, noise, tkey.tlwe_key)
    tgsw_add_message_seeded(thr, arr, m, tkey)
    body = arr.samples.a.coeffs[..., 1, :].contiguous().reshape(shape + (bits, 2, 2, N))
    return CompressedEncryptedIndexArray(params, shape, bits, seed, body, _variance(noise))


# ---------------------------------------------------------------- tables and lookups

def _table_shape(shape):
    """(W, m) of a table of shape (2^m,) or (W, 2^m), with the caps of the layout (ValueError otherwise)."""
    if len(shape) not in (1, 2) or (len(shape) == 2 and shape[0] < 1):
        raise ValueError('a table has shape (2^m,) or (W, 2^m), got %s' % (tuple(shape),))
    W, size = (1,) + tuple(shape) if len(shape) == 1 else tuple(shape)
    m = int(size).bit_length() - 1
    if size != 1 << m or not 1 <= m <= MAX_BITS:
        raise ValueError('a table has 2^m entries per column, 1 <= m <= %d, got %d' % (MAX_BITS, size))
    if m < ROTATE_BITS and W << m > N:
        raise ValueError('a table on %d index bits has at most %d columns, got %d' % (m, N >> m, W))
    return W, m


def _check_out(out, bits):
    if out not in ('int', 'bool'):
        raise ValueError("out must be 'int' or 'bool'")
    if out == 'int' and bits is None:
        raise ValueError("out='int' needs the message bits of the entries")


def table_polys_count(m, columns):
    """P, the GLWE samples of a table: W 2^(m-10) for m >= 10, else 1."""
    return columns << (m - ROTATE_BITS) if m >= ROTATE_BITS else 1


def _plain_layout(params, table, out, bits):
    """(single, W, m, plain): the entries of `table` encoded for `out` and laid out as (P, N) int32 plaintext
    polynomials (module docstring), 0 in the unused coefficients."""
    _check_params(params)
    _check_out(out, bits)
    table = numpy.asarray(table)
    W, m = _table_shape(table.shape)
    single = table.ndim == 1
    table = table.reshape(W, 1 << m)
    if out == 'int':
        enc = lut.encode_int(table, bits)
    else:
        enc = numpy.where(table != 0, int(MU), -int(MU)).astype(numpy.int32)
    plain = numpy.zeros((table_polys_count(m, W), N), numpy.int32)
    plain.reshape(-1)[:W << m] = enc.reshape(-1)
    return single, W, m, plain


class IndexTable:
    """W columns of 2^m entries encoded to Torus32 and laid out as GLWE plaintexts on the device (module docstring):
    `polys` (P, 2, N) int32 trivial samples (0, T), P = W 2^(m-10) for m >= 10, else 1.  out='int' encodes entries as
    `lut.encode_int(., bits)` (results feed vm.lut and decrypt_int), out='bool' as +-1/8 (results feed the gates)."""

    def __init__(self, thr, params, table, out='int', bits=None):
        self.single, W, m, plain = _plain_layout(params, table, out, bits)
        self.params = params
        self.out, self.bits_out = out, bits
        self.bits, self.columns = m, W
        polys = numpy.zeros((plain.shape[0], 2, N), numpy.int32)
        polys[:, 1] = plain
        self.polys = thr.to_device(polys)


class EncryptedIndexTable:
    """An IndexTable whose entries are encrypted: params, m (`bits`), W (`columns`), `out` / `bits_out` as IndexTable,
    the variance of the leaves' noise, the wire form `data` (P, 2, N) uint16 (mask and body rounded to 16 bits, 4 bytes
    per entry) and the device nodes `nodes` (P, 2, N) int32 = data << 16, laid out as IndexTable.polys.  Every leaf is a
    GLWE sample under the bootstrap key's GLWE key S whose phase carries the entry at its coefficient; unused
    coefficients encrypt 0.  Made by ctx.encrypt_table (client) or vm.make_encrypted_table (server); vm.lookup and
    mk.lookup take it where they take an IndexTable."""

    def __init__(self, thr, params, bits, columns, data, variance: float, out='int', bits_out=None, single=None):
        _check_params(params)
        _check_out(out, bits_out)
        W, m = _table_shape((int(columns), 1 << _check_bits(bits)))
        want = (table_polys_count(m, W), 2, N)
        if tuple(data.shape) != want or data.dtype != torch.uint16:
            raise ValueError('an encrypted table of %d columns on %d bits is uint16 %s, got %s %s'
                             % (W, m, want, data.dtype, tuple(data.shape)))
        self.params = params
        self.bits, self.columns = m, W
        self.out, self.bits_out = out, bits_out
        self.single = W == 1 if single is None else bool(single)
        self.variance = float(variance)
        self.data = data
        self.nodes = _wrap32((data.to(thr.device).view(torch.int16).to(torch.int64) & 0xffff) << 16).contiguous()

    def dump(self, file_obj):
        pickle.dump(_ENCRYPTED_TABLE_TAG, file_obj)
        for x in (self.params, self.bits, self.columns, self.single, self.out, self.bits_out, self.variance):
            pickle.dump(x, file_obj)
        pickle.dump(self.data.cpu().numpy().astype('<u2').tobytes(), file_obj)

    def dumps(self):
        file_obj = io.BytesIO()
        self.dump(file_obj)
        return file_obj.getvalue()

    @classmethod
    def load(cls, file_obj, thr):
        """ValueError for another pickle, a damaged one or data that does not fit the table's shape."""
        _check_tag(file_obj, _ENCRYPTED_TABLE_TAG)
        params, bits, columns, single, out, bits_out, variance, raw = compact._fields(file_obj, 8)
        W, m = _table_shape((int(columns), 1 << _check_bits(bits)))
        count = table_polys_count(m, W)
        if not isinstance(raw, bytes) or len(raw) != count * 2 * N * 2:
            raise ValueError('encrypted table data does not match %d columns on %d bits' % (W, m))
        data = numpy.frombuffer(raw, '<u2').astype(numpy.uint16).reshape(count, 2, N)
        return cls(thr, params, m, W, thr.to_device(data), variance, out, bits_out, single)

    @classmethod
    def loads(cls, s: bytes, thr):
        return cls.load(io.BytesIO(s), thr)

    def __eq__(self, other):
        return (self.__class__ == other.__class__ and self.params == other.params and self.bits == other.bits
                and self.columns == other.columns and self.single == other.single and self.out == other.out
                and self.bits_out == other.bits_out and self.variance == other.variance
                and numpy.array_equal(self.data.cpu().numpy(), other.data.cpu().numpy()))


def _round16(x):
    """int32 coefficients -> round(x / 2^16) mod 2^16 as uint16 (packing's rounding)."""
    u = ((x.to(torch.int64) & 0xffffffff) + 0x8000) >> 16
    return (u & 0xffff).to(torch.int32).to(torch.int16).view(torch.uint16)


def encrypt_table(thr, rng, key, table, out='int', bits=None):
    """An EncryptedIndexTable of `table` (shape (2^m,) or (W, 2^m), entries encoded and laid out as IndexTable does).
    With a NuFHECompactPublicKey, whoever holds it encrypts: compact_encrypt of the flattened layout, its draws.  With
    the owner's NuFHEIndexSecretKey: a GLWE encryption under S with tlwe_params.min_noise (draws the masks, then the
    noises, as tlwe_encrypt_zero), rounded to the same 16-bit form.  TypeError for any other key."""
    if isinstance(key, compact.NuFHECompactPublicKey):
        params = key.params
        single, W, m, plain = _plain_layout(params, table, out, bits)
        data = compact.compact_encrypt(thr, rng, key, thr.to_device(plain)).data
        fresh, mask_rnd, body_rnd, _ = compact.noise_terms(params)
        variance = fresh + mask_rnd + body_rnd
    elif isinstance(key, NuFHEIndexSecretKey):
        params = key.params
        single, W, m, plain = _plain_layout(params, table, out, bits)
        tl = params.tgsw_params.tlwe_params
        samples = TLweSampleArray.empty(thr, tl, (plain.shape[0],))
        tlwe_encrypt_zero(thr, rng, samples, tl.min_noise, key._tgsw_key().tlwe_key)
        x = samples.a.coeffs
        x[:, 1] = _wrap32((x[:, 1].to(torch.int64) + thr.to_device(plain).to(torch.int64)) & 0xffffffff)
        data = _round16(x)
        variance = tl.min_noise**2 + rounding_variance(params)
    else:
        raise TypeError('encrypt_table needs a NuFHECompactPublicKey or the NuFHEIndexSecretKey, got %s'
                        % type(key).__name__)
    return EncryptedIndexTable(thr, params, m, W, data, variance, out, bits, single)


def make_encrypted_table(thr, params, tree_key, columns, out='int', bits=None):
    """The EncryptedIndexTable whose entries are the LWE samples `columns` (an LweSampleArray of shape (2^m,) or
    (W, 2^m), or a list of W of shape (2^m,), under the cloud key's LWE key), packed under S with the tree key: the
    packing pipeline of DESIGN.md section 12 (packing.pack with the tree key's spectra), one GLWE sample per 1024 entries
    in the lookup layout.  The leaves carry the largest input variance, at least lut.bootstrap_variance, plus
    packing_variance.  TypeError unless tree_key is a NuFHETreeKey; ValueError for other parameters or a shape that is
    not a table's."""
    from .tree_lut import NuFHETreeKey
    if not isinstance(tree_key, NuFHETreeKey):
        raise TypeError('make_encrypted_table needs a NuFHETreeKey (ctx.make_cloud_key(sk, tree_key=True)), got %s'
                        % type(tree_key).__name__)
    if tree_key.params != params:
        raise ValueError('the tree key was made for other parameters than this virtual machine')
    _check_params(params)
    _check_out(out, bits)
    if out == 'int':
        lut._check_bits(bits)
    single = isinstance(columns, LweSampleArray) and len(columns.shape) == 1
    cols = [columns] if isinstance(columns, LweSampleArray) else list(columns)
    if not cols or not all(isinstance(c, LweSampleArray) for c in cols):
        raise TypeError('make_encrypted_table takes an LweSampleArray or a list of them')
    if any(c.params != params.in_out_params for c in cols):
        raise ValueError('the columns do not have the LWE parameters of this virtual machine')
    if len(cols) == 1:
        shape = tuple(cols[0].shape)
    elif all(len(c.shape) == 1 and tuple(c.shape) == tuple(cols[0].shape) for c in cols):
        shape = (len(cols),) + tuple(cols[0].shape)
    else:
        raise ValueError('a list of columns holds W arrays of one shape (2^m,)')
    W, m = _table_shape(shape)
    n = params.in_out_params.size
    flat = LweSampleArray(params.in_out_params, torch.cat([c.a.reshape(-1, n) for c in cols]),
                          torch.cat([c.b.reshape(-1) for c in cols]),
                          torch.cat([c.current_variances.reshape(-1) for c in cols]))
    data = packing.pack(thr, tree_key, flat).data         # W 2^m entries in C order: exactly the lookup layout
    # bootstrap outputs record the key switch's variance only (the blind rotation's is not tracked), so a leaf counts
    # at least a bootstrap output's estimate
    variance = max(float(flat.current_variances.max()), lut.bootstrap_variance(params)) + packing_variance(params)
    return EncryptedIndexTable(thr, params, m, W, data, variance, out, bits, single)


def _table_nodes(table):
    """The (P, 2, N) int32 leaves the first level reads, and the variance they carry."""
    if isinstance(table, EncryptedIndexTable):
        return table.nodes, table.variance
    return table.polys, 0.0


def queries_per_pass(m, columns, tables=0):
    """Queries per pass of `lookup`: as many as keep the selector spectra, the tree nodes and `tables` concatenated
    encrypted tables (mk.lookup with one table per tenant: 8 MB each at m = 20) within PASS_BYTES."""
    spectra = m * 16 * 512 * 16                                     # BK_FFT_U64 words of 8 bytes per bit
    nodes = (columns << max(m - ROTATE_BITS, 0)) * NODE_BYTES if m > ROTATE_BITS else 0
    table_bytes = tables * table_polys_count(m, columns) * NODE_BYTES
    return max(1, (PASS_BYTES - table_bytes) // (spectra + nodes))


def selector_passes(thr, m, W, sels, per_tenant=False):
    """The passes of a batch of queries (selector arrays (c, m, 2, 2, 2, N), one per tenant, in order) that lookups and
    writes share: yields q0, q1, the tenants owning queries [q0, q1) and how many each owns, and the selector spectra
    (q1 - q0, m, R) of those queries.  With `per_tenant` a pass leaves room for one table per tenant it serves."""
    counts = [s.shape[0] for s in sels]
    starts = numpy.cumsum([0] + counts)
    B = int(starts[-1])
    q0 = 0
    while q0 < B:
        if not per_tenant:
            step = queries_per_pass(m, W)
        else:           # as many queries as leave room for the tables of the tenants they belong to
            k = 1
            while True:
                step = queries_per_pass(m, W, k)
                k2 = len(owners(counts, q0, min(B, q0 + step))[0])
                if k2 <= k:
                    break
                k = k2
        q1 = min(B, q0 + step)
        Q = q1 - q0
        idx, own = owners(counts, q0, q1) if len(sels) > 1 else ([0], [Q])
        pieces = [sels[i][max(q0, starts[i]) - starts[i]:][:c] for i, c in zip(idx, own)]
        spec = thr.index_prepare(torch.cat(pieces) if len(pieces) > 1 else pieces[0]).reshape(Q, m, -1)
        yield q0, q1, idx, own, spec
        del spec, pieces            # one pass's spectra on the device at a time
        q0 = q1


def lookup_passes(thr, m, W, sels, table=None, tables=None):
    """The lookup_extracted samples of the queries of `sels` (selector arrays (c, m, 2, 2, 2, N), one per tenant, in
    order) a pass at a time: yields q0, q1 and a (W, q1 - q0, N), b (W, q1 - q0) of queries [q0, q1).  Every query reads
    `table`, or, with `tables` (one EncryptedIndexTable per tenant), its tenant's table from the first level on."""
    for q0, q1, idx, own, spec in selector_passes(thr, m, W, sels, tables is not None):
        Q = q1 - q0
        j0 = ROTATE_BITS
        cur = _table_nodes(table)[0] if tables is None else None    # shared by every query until the first CMux level
        if tables is not None:
            # the pass's distinct tables, concatenated, and the table of every query
            uniq = {}
            slot = [uniq.setdefault(id(tables[i]), (len(uniq), tables[i]))[0] for i in idx]
            nodes = torch.cat([tb.nodes for _, tb in uniq.values()]) if len(uniq) > 1 else tables[idx[0]].nodes
            nodes = nodes.reshape(len(uniq), -1, 2, N)
            ids = numpy.repeat(numpy.asarray(slot, numpy.uint32), own)
            if m > j0:
                cur, j0 = thr.index_cmux_level_indirect(nodes, ids, spec, j0, Q), j0 + 1
            else:
                a, b = thr.index_rotate_extract_indirect(nodes, ids, spec, m, W, Q)
            del nodes
        if cur is not None:
            for j in range(j0, m):
                cur = thr.index_cmux_level(cur, spec, j, Q)
            a, b = thr.index_rotate_extract(cur, spec, m, W, Q)
        del spec, cur
        yield q0, q1, a, b


def lookup_extracted(thr, index, table):
    """The lookup before the key switch: LWE samples under the N-word key of S, a (W, B, N) and b (W, B) int32 for the
    B = prod(index.shape) queries, column w of query q at [w, q]."""
    m, W = table.bits, table.columns
    B = int(numpy.prod(index.shape, dtype=numpy.int64))
    out_a, out_b = thr.empty((W, B, N), torch.int32), thr.empty((W, B), torch.int32)
    for q0, q1, a, b in lookup_passes(thr, m, W, [index.samples.reshape(B, m, 2, 2, 2, N)], table):
        if q1 - q0 == B:
            return a, b
        out_a[:, q0:q1] = a
        out_b[:, q0:q1] = b
    return out_a, out_b


def lookup(thr, ks, index, table, dest=None):
    """table[idx] for every encrypted index of `index`: a list of W LweSampleArrays of the index's shape under the
    user's key (one array for a one-dimensional table).  TypeError unless `index` is an EncryptedIndexArray (a
    compressed one must be decompressed first) and `table` an IndexTable or EncryptedIndexTable; ValueError for other
    parameters or an index bit count that is not the table's m.  The results' variances add an encrypted table's leaf
    variance: a CMux passes the selected leaf's noise through unchanged."""
    if not isinstance(index, EncryptedIndexArray):
        raise TypeError('lookup needs an EncryptedIndexArray%s, got %s'
                        % (' (decompress() it first)' if isinstance(index, CompressedEncryptedIndexArray) else '',
                           type(index).__name__))
    if not isinstance(table, (IndexTable, EncryptedIndexTable)):
        raise TypeError('lookup needs an IndexTable (vm.make_index_table) or an EncryptedIndexTable, got %s'
                        % type(table).__name__)
    if index.params != table.params:
        raise ValueError('the encrypted index was made for other parameters than this table')
    if index.bits != table.bits:
        raise ValueError('the table takes %d-bit indices, got %d bits' % (table.bits, index.bits))
    params = table.params
    W = table.columns
    shape = index.shape
    B = int(numpy.prod(shape, dtype=numpy.int64))
    n = params.in_out_params.size
    if dest is None:
        dest = [LweSampleArray.empty(thr, params.in_out_params, shape) for _ in range(W)]
    elif isinstance(dest, LweSampleArray):
        dest = [dest]
    if len(dest) != W or any(tuple(d.shape) != shape for d in dest):
        raise ValueError('lookup writes %d results of shape %s' % (W, shape))
    a, b = lookup_extracted(thr, index, table)
    ra, rb, _ = thr.keyswitch(ks.device_arrays(), (a.reshape(W * B, N), b.reshape(W * B)))
    ra, rb = ra.reshape(W, B, n), rb.reshape(W, B)
    for w, r in enumerate(dest):
        r.a.copy_(ra[w].reshape(shape + (n,)))
        r.b.copy_(rb[w].reshape(shape))
        r.current_variances.fill_(float(_table_nodes(table)[1] + output_variance(params, table.bits)))
    return dest[0] if table.single else dest
