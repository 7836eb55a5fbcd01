"""Low-level API (reference: nufhe/api_low_level.py)."""
import io
import pickle

import numpy

from .numeric_functions import phase_to_t32
from .lwe import LweParams, LweKey, LweSampleArray, lwe_encrypt, lwe_decrypt, LweKeyswitchKey
from .tgsw import TGswParams, TGswKey
from .tlwe import TLweParams
from .bootstrap import BootstrapKey, MultiBitBootstrapKey, check_multi_bit
from .performance import PerformanceParameters, PerformanceParametersForDevice


class NuFHEParameters:
    """Parameters of the FHE scheme (api_low_level.py:31-87).

    :param transform_type: only ``'NTT'`` is built here (the integer, bit-exact transform);
        ``'FFT'`` raises ``ValueError``.
    :param tlwe_mask_size: the TLWE mask size k.  1 (default) runs on the fused bootstrap kernel; larger values run
        on the multi-kernel path, like in the reference (its single-kernel path has the same limit,
        blind_rotate.py:53-58).
    """

    def __init__(self, transform_type='NTT', tlwe_mask_size=1):
        assert transform_type in ('FFT', 'NTT')
        assert tlwe_mask_size >= 1
        if transform_type != 'NTT':
            raise ValueError("nufhe_b200 implements the NTT transform only")

        tlwe_polynomial_degree = 1024
        lwe_size = 500
        bs_decomp_length = 2
        bs_log2_base = 10
        ks_decomp_length = 8
        ks_log2_base = 2
        coeff = (2 / numpy.pi)**0.5
        ks_stdev = 1 / 2**15 * coeff
        bs_stdev = 9e-9 * coeff
        max_stdev = 1 / 2**4 / 4 * coeff

        params_in = LweParams(lwe_size, ks_stdev, max_stdev)
        params_accum = TLweParams(tlwe_polynomial_degree, tlwe_mask_size, bs_stdev, max_stdev, transform_type)
        params_bs = TGswParams(params_accum, bs_decomp_length, bs_log2_base)

        self.ks_decomp_length = ks_decomp_length
        self.ks_log2_base = ks_log2_base
        self.in_out_params = params_in
        self.tgsw_params = params_bs
        self._transform_type = transform_type
        self._tlwe_mask_size = tlwe_mask_size

    def __hash__(self):
        return hash((self.__class__, self._transform_type, self._tlwe_mask_size))

    def __eq__(self, other):
        return (self.__class__ == other.__class__ and self._transform_type == other._transform_type
                and self._tlwe_mask_size == other._tlwe_mask_size)


class NuFHESecretKey:
    """api_low_level.py:90-154"""

    def __init__(self, params: NuFHEParameters, lwe_key: LweKey):
        self.params = params
        self.lwe_key = lwe_key

    @classmethod
    def from_rng(cls, thr, params: NuFHEParameters, rng):
        return cls(params, LweKey.from_rng(thr, params.in_out_params, rng))

    def dump(self, file_obj):
        pickle.dump(self.params, file_obj)
        self.lwe_key.dump(file_obj)

    def dumps(self):
        file_obj = io.BytesIO()
        self.dump(file_obj)
        return file_obj.getvalue()

    @classmethod
    def load(cls, file_obj, thr):
        params = pickle.load(file_obj)
        return cls(params, LweKey.load(file_obj, thr))

    @classmethod
    def loads(cls, s: bytes, thr):
        return cls.load(io.BytesIO(s), thr)

    def __eq__(self, other):
        return (self.__class__ == other.__class__ and self.params == other.params
                and self.lwe_key == other.lwe_key)


class NuFHECloudKey:
    """api_low_level.py:157-239"""

    def __init__(self, params: NuFHEParameters, bootstrap_key: BootstrapKey, keyswitch_key: LweKeyswitchKey):
        self.params = params
        self.bootstrap_key = bootstrap_key
        self.keyswitch_key = keyswitch_key

    @classmethod
    def from_rng(cls, thr, params: NuFHEParameters, rng, secret_key: NuFHESecretKey,
                 perf_params: PerformanceParametersForDevice = None):
        return cls.from_rng_with_tgsw_key(thr, params, rng, secret_key, perf_params)[0]

    @classmethod
    def from_rng_with_tgsw_key(cls, thr, params: NuFHEParameters, rng, secret_key: NuFHESecretKey,
                               perf_params: PerformanceParametersForDevice = None, multi_bit=1):
        """(cloud key, TGswKey): the TGSW key, which from_rng discards, is what a tree key is made with.
        multi_bit=2 makes a MultiBitBootstrapKey in the bootstrap key's place (bootstrap.py)."""
        check_multi_bit(params, multi_bit)
        if perf_params is None:
            perf_params = PerformanceParameters(params).for_device(thr.device_params)
        tgsw_key = TGswKey.from_rng(thr, params.tgsw_params, rng)
        bk_cls = MultiBitBootstrapKey if multi_bit == 2 else BootstrapKey
        bk = bk_cls.from_rng(thr, rng, secret_key.lwe_key, tgsw_key, perf_params)
        ks = LweKeyswitchKey.from_tgsw_key(
            thr, rng, params.ks_decomp_length, params.ks_log2_base, secret_key.lwe_key, tgsw_key)
        return cls(params, bk, ks), tgsw_key

    def dump(self, file_obj):
        pickle.dump(self.params, file_obj)
        self.bootstrap_key.dump(file_obj)
        self.keyswitch_key.dump(file_obj)

    def dumps(self):
        file_obj = io.BytesIO()
        self.dump(file_obj)
        return file_obj.getvalue()

    @classmethod
    def load(cls, file_obj, thr):
        params = pickle.load(file_obj)
        bootstrap_key = BootstrapKey.load(file_obj, thr)
        keyswitch_key = LweKeyswitchKey.load(file_obj, thr)
        return cls(params, bootstrap_key, keyswitch_key)

    @classmethod
    def loads(cls, s: bytes, thr):
        return cls.load(io.BytesIO(s), thr)

    def __eq__(self, other):
        return (self.__class__ == other.__class__ and self.params == other.params
                and self.bootstrap_key == other.bootstrap_key
                and self.keyswitch_key == other.keyswitch_key)


def make_key_pair(thr, rng, **params):
    """api_low_level.py:242-250"""
    nufhe_params = NuFHEParameters(**params)
    secret_key = NuFHESecretKey.from_rng(thr, nufhe_params, rng)
    cloud_key = NuFHECloudKey.from_rng(thr, nufhe_params, rng, secret_key)
    return secret_key, cloud_key


_1s8 = phase_to_t32(1, 8)


def bool_to_t32(bits):
    return numpy.where(numpy.asarray(bits).astype(bool), _1s8, -_1s8).astype(numpy.int32)


def t32_to_bool(mu):
    return numpy.asarray(mu) > 0


def _encrypt_mus(thr, rng, key, shape, mus, compressed):
    from .public_key import NuFHEPublicKey, public_encrypt
    from .compact import NuFHECompactPublicKey, compact_encrypt
    if isinstance(key, NuFHECompactPublicKey):
        if compressed:
            raise ValueError("a compact public-key encryption is already compact: compressed=True does not apply")
        return compact_encrypt(thr, rng, key, mus.reshape(shape))
    if isinstance(key, NuFHEPublicKey):
        if compressed:
            raise ValueError("a public-key encryption cannot be compressed: its mask depends on the secret random "
                             "matrix R, not on a seed that can be published")
        return public_encrypt(thr, rng, key, mus.reshape(shape))
    noise = key.params.in_out_params.min_noise
    if compressed:
        from .compressed import CompressedLweSampleArray
        return CompressedLweSampleArray.encrypt(thr, rng, key.params.in_out_params, mus.reshape(shape), noise,
                                                key.lwe_key)
    result = empty_ciphertext(thr, key.params, shape)
    lwe_encrypt(thr, rng, result, mus, noise, key.lwe_key)
    return result


def encrypt(thr, rng, key, message, compressed=False):
    """api_low_level.py:266-281.  compressed=True returns a CompressedLweSampleArray: the mask is regenerated from a
    seed (nufhe_b200/compressed.py), so only the bodies and the seed are stored or sent.  `key` is a NuFHESecretKey or
    a NuFHEPublicKey (nufhe_b200/public_key.py; not with compressed=True); a NuFHECompactPublicKey
    (nufhe_b200/compact.py; not with compressed=True) gives a CompactLweSampleArray."""
    message = numpy.asarray(message)
    mus = thr.to_device(numpy.ascontiguousarray(bool_to_t32(message)))
    return _encrypt_mus(thr, rng, key, message.shape, mus, compressed)


def decrypt(thr, key: NuFHESecretKey, ciphertext: LweSampleArray):
    """api_low_level.py:284-295"""
    mus = lwe_decrypt(thr, ciphertext, key.lwe_key)
    return t32_to_bool(mus)


def encrypt_int(thr, rng, key, values, bits, compressed=False):
    """Encrypt integers in [0, 2^bits), bits = 1..3, for lookup tables (nufhe_b200/lut.py: m * 2^(31 - bits)).
    compressed=True returns a CompressedLweSampleArray, as for encrypt(); `key` may be a NuFHEPublicKey or a
    NuFHECompactPublicKey."""
    from .lut import encode_int
    values = numpy.asarray(values)
    mus = thr.to_device(numpy.ascontiguousarray(encode_int(values, bits)))
    return _encrypt_mus(thr, rng, key, values.shape, mus, compressed)


def decrypt_int(thr, key: NuFHESecretKey, ciphertext: LweSampleArray, bits):
    """The integers in [0, 2^bits) that `ciphertext` holds (encrypt_int's encoding)."""
    from .lut import decode_int
    return decode_int(lwe_decrypt(thr, ciphertext, key.lwe_key), bits)


def empty_ciphertext(thr, params: NuFHEParameters, shape):
    """api_low_level.py:298-302"""
    return LweSampleArray.empty(thr, params.in_out_params, tuple(shape))
