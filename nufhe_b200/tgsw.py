"""TGSW parameters, keys and the bootstrap-key container (reference: nufhe/tgsw.py)."""
import pickle

import numpy
import torch

from .numeric_functions import Torus32
from .tlwe import (
    TLweParams, TLweKey, TLweSampleArray, TransformedTLweSampleArray,
    tlwe_transform_samples, tlwe_encrypt_zero)


class TGswParams:
    """tgsw.py:43-67"""

    def __init__(self, tlwe_params: TLweParams, decomp_length: int, bs_log2_base: int):
        decomp_range = numpy.arange(1, decomp_length + 1)
        self.base_powers = (2**(32 - decomp_range * bs_log2_base)).astype(Torus32)
        offset = int(self.base_powers.astype(numpy.int64).sum() * (2**bs_log2_base // 2))
        self.offset = Torus32(offset - 2**32 if offset >= 2**31 else offset)
        self.decomp_length = decomp_length
        self.bs_log2_base = bs_log2_base
        self.tlwe_params = tlwe_params

    def __eq__(self, other):
        return (self.__class__ == other.__class__ and self.decomp_length == other.decomp_length
                and self.bs_log2_base == other.bs_log2_base and self.tlwe_params == other.tlwe_params)

    def __hash__(self):
        return hash((self.__class__, self.decomp_length, self.bs_log2_base, self.tlwe_params))


class TGswKey:
    def __init__(self, params: TGswParams, tlwe_key: TLweKey):
        self.params = params
        self.tlwe_key = tlwe_key

    @classmethod
    def from_rng(cls, thr, params: TGswParams, rng):
        return cls(params, TLweKey.from_rng(thr, params.tlwe_params, rng))


class TGswSampleArray:
    """tgsw.py:81-96"""

    def __init__(self, params: TGswParams, samples: TLweSampleArray):
        self.mask_size = params.tlwe_params.mask_size
        self.decomp_length = params.decomp_length
        self.samples = samples
        self.params = params
        self.shape = samples.shape[:-2]

    @classmethod
    def empty(cls, thr, params: TGswParams, shape):
        k = params.tlwe_params.mask_size
        samples = TLweSampleArray.empty(
            thr, params.tlwe_params, tuple(shape) + (k + 1, params.decomp_length))
        return cls(params, samples)


class TransformedTGswSampleArray:
    """tgsw.py:99-130.  samples.a.coeffs: (n, k+1, l, k+1, N) uint64 (as int64 bits), natural NTT order,
    Montgomery form -- the reference's bootstrap-key wire format."""

    def __init__(self, params: TGswParams, samples: TransformedTLweSampleArray):
        self.mask_size = params.tlwe_params.mask_size
        self.decomp_length = params.decomp_length
        self.samples = samples
        self.params = params
        self.shape = samples.shape[:-2]

    @classmethod
    def empty(cls, thr, params: TGswParams, shape):
        k = params.tlwe_params.mask_size
        samples = TransformedTLweSampleArray.empty(
            thr, params.tlwe_params, tuple(shape) + (k + 1, params.decomp_length))
        return cls(params, samples)

    def dump(self, file_obj):
        pickle.dump(self.params, file_obj)
        self.samples.dump(file_obj)

    @classmethod
    def load(cls, file_obj, thr):
        params = pickle.load(file_obj)
        samples = TransformedTLweSampleArray.load(file_obj, thr)
        return cls(params, samples)

    def __eq__(self, other):
        return (self.__class__ == other.__class__ and self.params == other.params
                and self.samples == other.samples)


def tgsw_transform_samples(thr, result: TransformedTGswSampleArray, source: TGswSampleArray, perf_params=None):
    tlwe_transform_samples(thr, result.samples, source.samples, perf_params)


def tgsw_add_message(thr, result: TGswSampleArray, messages):
    """TGswAddMessage (tgsw_gpu.py:172-205, tgsw_gpu.mako:18-39; ref tgsw_cpu.py:109-126):
    result += message * H, i.e. += m * 2^(32-10(j+1)) at [.., mi, j, mi, 0]."""
    params = result.params
    k = params.tlwe_params.mask_size
    coeffs = result.samples.a.coeffs
    base_powers = torch.from_numpy(params.base_powers.astype(numpy.int64)).to(coeffs.device)
    inc = messages.to(torch.int64).reshape(-1, 1) * base_powers.reshape(1, -1)
    view = coeffs.reshape((-1,) + tuple(coeffs.shape[-4:]))
    for mi in range(k + 1):
        v = (view[:, mi, :, mi, 0].to(torch.int64) + inc) & 0xffffffff
        view[:, mi, :, mi, 0] = torch.where(v >= 2**31, v - 2**32, v).to(torch.int32)


def tgsw_encrypt_zero(thr, rng, result: TGswSampleArray, noise: float, key: TGswKey, perf_params=None):
    tlwe_encrypt_zero(thr, rng, result.samples, noise, key.tlwe_key, perf_params)


def tgsw_encrypt_int(thr, rng, result: TGswSampleArray, messages, noise: float, key: TGswKey, perf_params=None):
    """tgsw.py:153-161"""
    tgsw_encrypt_zero(thr, rng, result, noise, key, perf_params)
    tgsw_add_message(thr, result, messages)


def fused_kernel_supported(params: TGswParams):
    """The parameter set of the fused bootstrap kernel (the reference's single-kernel path has the same limits,
    blind_rotate.py:37-86)."""
    return (params.tlwe_params.mask_size == 1 and params.decomp_length == 2 and params.bs_log2_base == 10
            and params.tlwe_params.polynomial_degree == 1024)


def tgsw_transformed_external_mul_steps(thr, result: TLweSampleArray, bootstrap_key, bk_row_idx: int):
    """The external product as the reference's computation composes it (tgsw_gpu.py:110-169): gadget decomposition,
    forward transforms, multiply-accumulate with the key row in the reference's own layout, inverse transforms.
    Works for any TLWE mask size k and decomposition length."""
    params = bootstrap_key.params
    k, l = params.tlwe_params.mask_size, params.decomp_length
    coeffs = result.a.coeffs
    dec = thr.tgsw_decompose(coeffs, l, params.bs_log2_base, params.offset)          # (..., k+1, l, N)
    tr = thr.ntt_forward_i32(dec)
    row = bootstrap_key.samples.a.coeffs[bk_row_idx]                                 # (k+1, l, k+1, N)
    mac = thr.tgsw_mac(tr, row, k, l)
    res = thr.ntt_inverse_i32(mac)
    coeffs.copy_(res.reshape(coeffs.shape))


def tgsw_transformed_external_mul(thr, result: TLweSampleArray, bootstrap_key, bk_row_idx: int, perf_params=None):
    """tgsw.py:165-172: result <- bootstrap_key[bk_row_idx] (x) result.
    `bootstrap_key` is a BootstrapKey-owned TransformedTGswSampleArray.  For the default parameters (k = 1, l = 2)
    this is one launch of the fused kernel's step on the engine-format copy of the key (built once, cached); any
    other mask size / decomposition goes through the separate steps above."""
    assert len(bootstrap_key.shape) == 1
    if not fused_kernel_supported(bootstrap_key.params):
        tgsw_transformed_external_mul_steps(thr, result, bootstrap_key, bk_row_idx)
        return
    bk_int = engine_format(thr, bootstrap_key)
    coeffs = result.a.coeffs
    if coeffs.is_contiguous():
        thr.external_product(coeffs, bk_int, bk_row_idx)
    else:
        tmp = coeffs.contiguous()
        thr.external_product(tmp, bk_int, bk_row_idx)
        coeffs.copy_(tmp)


def engine_format(thr, tgsw: TransformedTGswSampleArray):
    """The bootstrap key re-laid for the MAC stage of the fused kernel (nb_bk_prepare, or nb_bk_prepare_multibit for
    the rows of a multi-bit key), cached."""
    if not fused_kernel_supported(tgsw.params):
        raise ValueError("The fused bootstrap kernel supports mask_size=1, decomp_length=2, bs_log2_base=10, "
                         "polynomial_degree=1024 only; other parameters run on the multi-kernel path "
                         "(single_kernel_bootstrap=False)")
    cached = getattr(tgsw, '_engine_format', None)
    if cached is None or cached.device != tgsw.samples.a.coeffs.device:
        if getattr(tgsw, 'multi_bit', 1) == 2:
            cached = thr.bk_prepare_multibit(tgsw.samples.a.coeffs)     # bootstrap.py: MultiBitBootstrapKey
        else:
            cached = thr.bk_prepare(tgsw.samples.a.coeffs)
        tgsw._engine_format = cached
    return cached
