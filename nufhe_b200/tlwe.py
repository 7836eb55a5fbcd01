"""Torus LWE containers and key-generation helpers (reference: nufhe/tlwe.py)."""
import pickle

import numpy
import torch

from . import _native
from .utils import arrays_equal
from .lwe import LweParams
from .polynomials import TorusPolynomialArray, IntPolynomialArray, TransformedPolynomialArray
from .random_numbers import rand_uniform_bool, rand_gaussian_torus32, rand_uniform_torus32


class TLweParams:
    """tlwe.py:48-75"""

    def __init__(self, polynomial_degree: int, mask_size: int, min_noise: float, max_noise: float,
                 transform_type):
        self.polynomial_degree = polynomial_degree
        self.mask_size = mask_size
        self.min_noise = min_noise
        self.max_noise = max_noise
        self.extracted_lweparams = LweParams(polynomial_degree * mask_size, min_noise, max_noise)
        self.transform_type = transform_type

    def __eq__(self, other):
        return (self.__class__ == other.__class__
                and self.polynomial_degree == other.polynomial_degree
                and self.mask_size == other.mask_size and self.min_noise == other.min_noise
                and self.max_noise == other.max_noise and self.transform_type == other.transform_type)

    def __hash__(self):
        return hash((self.__class__, self.polynomial_degree, self.mask_size, self.min_noise,
                     self.max_noise, self.transform_type))


class TLweKey:
    """tlwe.py:78-92"""

    def __init__(self, params: TLweParams, key):
        self.params = params
        self.key = key

    @classmethod
    def from_rng(cls, thr, params: TLweParams, rng):
        key = IntPolynomialArray(
            rand_uniform_bool(thr, rng, (params.mask_size, params.polynomial_degree)))
        return cls(params, key)


class TLweSampleArray:
    """tlwe.py:94-113: a.coeffs has shape `shape + (k+1, N)`"""

    def __init__(self, params: TLweParams, a, current_variances):
        self.a = a
        self.current_variances = current_variances
        self.shape = tuple(current_variances.shape)
        self.params = params

    @classmethod
    def empty(cls, thr, params: TLweParams, shape):
        shape = tuple(shape)
        a = TorusPolynomialArray.empty(thr, params.polynomial_degree, shape + (params.mask_size + 1,))
        current_variances = torch.zeros(shape, dtype=torch.float32, device=thr.device)
        return cls(params, a, current_variances)


class TransformedTLweSampleArray:
    """tlwe.py:115-152"""

    def __init__(self, params: TLweParams, a, current_variances):
        self.a = a
        self.current_variances = current_variances
        self.shape = tuple(current_variances.shape)
        self.params = params

    @classmethod
    def empty(cls, thr, params: TLweParams, shape):
        shape = tuple(shape)
        a = TransformedPolynomialArray.empty(
            thr, params.transform_type, params.polynomial_degree, shape + (params.mask_size + 1,))
        current_variances = torch.zeros(shape, dtype=torch.float32, device=thr.device)
        return cls(params, a, current_variances)

    def dump(self, file_obj):
        pickle.dump(self.params, file_obj)
        self.a.dump(file_obj)
        pickle.dump(self.current_variances.cpu().numpy(), file_obj)

    @classmethod
    def load(cls, file_obj, thr):
        params = pickle.load(file_obj)
        a = TransformedPolynomialArray.load(file_obj, thr)
        current_variances = pickle.load(file_obj)
        return cls(params, a, thr.to_device(current_variances))

    def __eq__(self, other):
        return (self.__class__ == other.__class__ and self.params == other.params
                and self.a == other.a
                and arrays_equal(self.current_variances, other.current_variances))


def tlwe_encrypt_zero(thr, rng, result: TLweSampleArray, noise: float, key: TLweKey, perf_params=None):
    """tlwe.py:184-197 -> TLweEncryptZero (tlwe_gpu.py:111-196; ref tlwe_cpu.py:64-89):
    mask = uniform, body = gaussian + sum_i key_i * mask_i, the product taken through the NTT
    (forward, field multiply, inverse) exactly like the reference's computation."""
    N = key.params.polynomial_degree
    k = key.params.mask_size
    noises1 = rand_uniform_torus32(thr, rng, result.shape + (k, N))
    noises2 = rand_gaussian_torus32(thr, rng, 0, noise, result.shape + (N,))
    tlwe_encrypt_zero_with_masks(thr, result, noises1, noises2, noise, key)


def tlwe_encrypt_zero_with_masks(thr, result: TLweSampleArray, noises1, noises2, noise: float, key: TLweKey):
    """tlwe_encrypt_zero with given masks `noises1` (shape + (k, N)) and body noises `noises2` (shape + (N,)); draws
    nothing.  Compressed bootstrap keys pass masks expanded from a seed (nufhe_b200/compressed.py)."""
    k = key.params.mask_size
    tr_key = thr.ntt_forward_i32(key.key.coeffs)                     # (k, N)
    tr_noise = thr.ntt_forward_i32(noises1)                          # shape + (k, N)
    prod = thr.ff_op(_native.FF_MUL, tr_noise, tr_key)               # key broadcast with period k*N
    conv = thr.ntt_inverse_i32(prod)                                 # shape + (k, N)
    body = noises2.contiguous()                                      # Torus32 wrap-around sums on the engine (nb_tlwe_add_to)
    for i in range(k):
        thr.tlwe_add_to(body, conv[..., i, :].contiguous())
    result.a.coeffs[..., :k, :] = noises1
    result.a.coeffs[..., k, :] = body
    result.current_variances.fill_(float(numpy.float32(noise**2)))


def tlwe_transform_samples(thr, result: TransformedTLweSampleArray, source: TLweSampleArray, perf_params=None):
    """tlwe.py:200-207 -> TLweTransformSamples (tlwe_gpu.py:199-236): forward NTT, then Montgomery form."""
    tr = thr.ntt_forward_i32(source.a.coeffs)
    result.a.coeffs.copy_(thr.ff_op(_native.FF_PREPARE, tr))
    result.current_variances.copy_(source.current_variances)


def tlwe_noiseless_trivial(thr, result: TLweSampleArray, mu: TorusPolynomialArray):
    """result = (0, mu) (tlwe.py:156-158, K8)."""
    thr.tlwe_noiseless_trivial(result.a.coeffs, result.current_variances, mu.coeffs)


def tlwe_extract_lwe_samples(thr, result, x: TLweSampleArray):
    """Sample extraction (tlwe.py:161-165, K9); `current_variances` of the result is left alone like the reference."""
    if result.a.is_contiguous() and result.b.is_contiguous():
        thr.tlwe_extract_lwe_samples(result.a, result.b, x.a.coeffs)
    else:
        a, b = torch.empty_like(result.a, memory_format=torch.contiguous_format), torch.empty_like(
            result.b, memory_format=torch.contiguous_format)
        thr.tlwe_extract_lwe_samples(a, b, x.a.coeffs)
        result.a.copy_(a)
        result.b.copy_(b)


def tlwe_shift_polynomials(thr, result: TLweSampleArray, bk: TLweSampleArray, powers, powers_idx):
    """result = (X^powers[.., powers_idx] - 1) * bk (tlwe.py:168-169)."""
    from .polynomials import shift_tp_minus_one_power_from_array
    shift_tp_minus_one_power_from_array(thr, result.a, powers, powers_idx, bk.a)


def tlwe_add_to(thr, result: TLweSampleArray, source: TLweSampleArray):
    """result += source (tlwe.py:173-175)."""
    thr.tlwe_add_to(result.a.coeffs, source.a.coeffs, result.current_variances, source.current_variances)


def tlwe_copy(thr, result: TLweSampleArray, source: TLweSampleArray):
    """result = source (tlwe.py:178-180; coefficients only, like the reference)."""
    result.a.coeffs.copy_(source.a.coeffs)
