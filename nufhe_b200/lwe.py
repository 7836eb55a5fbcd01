"""LWE containers and operations (reference: nufhe/lwe.py).

Device arrays are torch CUDA tensors: `a` (shape + (n,)) int32, `b` (shape) int32,
`current_variances` (shape) float32, C-contiguous or NumPy-style views of such (lwe.py:152-172).
`thr` is a nufhe_b200.engine.Engine (the analogue of a Reikna Thread)."""
import io
import pickle

import numpy
import torch

from .utils import arrays_equal
from .numeric_functions import Torus32, ErrorFloat
from .random_numbers import rand_uniform_bool, rand_uniform_torus32, rand_gaussian_torus32


class LweParams:
    """lwe.py:53-68"""

    def __init__(self, size: int, min_noise: float, max_noise: float):
        self.size = size
        self.min_noise = min_noise
        self.max_noise = max_noise

    def __eq__(self, other):
        return (self.__class__ == other.__class__ and self.size == other.size
                and self.min_noise == other.min_noise and self.max_noise == other.max_noise)

    def __hash__(self):
        return hash((self.__class__, self.size, self.min_noise, self.max_noise))


class LweKey:
    """lwe.py:71-106"""

    def __init__(self, params: LweParams, key):
        self.params = params
        self.key = key

    @classmethod
    def from_rng(cls, thr, params: LweParams, rng):
        return cls(params, rand_uniform_bool(thr, rng, (params.size,)))

    @classmethod
    def from_tlwe_key(cls, params: LweParams, tlwe_key):
        assert params.size == tlwe_key.params.polynomial_degree * tlwe_key.params.mask_size
        return cls(params, tlwe_key.key.coeffs.reshape(-1))

    def dump(self, file_obj):
        pickle.dump(self.params, file_obj)
        pickle.dump(self.key.cpu().numpy(), file_obj)

    @classmethod
    def load(cls, file_obj, thr):
        params = pickle.load(file_obj)
        key = pickle.load(file_obj)
        return cls(params, thr.to_device(key))

    def __eq__(self, other):
        return (self.__class__ == other.__class__ and self.params == other.params
                and arrays_equal(self.key, other.key))


class LweSampleArrayShapeInfo:
    """lwe.py:109-132 (shapes and strides are what the reference's compile cache keys on)."""

    def __init__(self, a, b, current_variances):
        if (not (len(a.shape) - 1 == len(b.shape) == len(current_variances.shape))
                or not (tuple(a.shape[:-1]) == tuple(b.shape) == tuple(current_variances.shape))):
            raise ValueError("Inconsistent shapes: {a}, {b}, {cv}".format(
                a=tuple(a.shape), b=tuple(b.shape), cv=tuple(current_variances.shape)))
        self.a = (tuple(a.shape), tuple(a.stride()))
        self.b = (tuple(b.shape), tuple(b.stride()))
        self.current_variances = (tuple(current_variances.shape), tuple(current_variances.stride()))
        self.shape = tuple(b.shape)

    def __eq__(self, other):
        return (self.__class__ == other.__class__ and self.a == other.a and self.b == other.b
                and self.current_variances == other.current_variances)

    def __hash__(self):
        return hash((self.__class__, self.a, self.b, self.current_variances))


class LweSampleArray:
    """A ciphertext object (lwe.py:135-251).  `shape` is the shape of the encrypted message."""

    def __init__(self, params: LweParams, a, b, current_variances):
        self.params = params
        self.a = a
        self.b = b
        self.current_variances = current_variances
        self.shape_info = LweSampleArrayShapeInfo(a, b, current_variances)

    @classmethod
    def empty(cls, thr, params: LweParams, shape):
        shape = tuple(shape)
        a = thr.empty(shape + (params.size,), torch.int32)
        b = thr.empty(shape, torch.int32)
        current_variances = thr.empty(shape, torch.float32)
        return cls(params, a, b, current_variances)

    @property
    def shape(self):
        return self.shape_info.shape

    def _a_index(self, index):
        """The message-shape index applied to `a`, whose last axis is the LWE dimension: an Ellipsis must
        not swallow that axis."""
        idx = index if isinstance(index, tuple) else (index,)
        if any(i is Ellipsis for i in idx):
            pos = [k for k, i in enumerate(idx) if i is Ellipsis][0]
            consumed = sum(1 for i in idx if i is not Ellipsis and i is not None)
            fill = (slice(None),) * (len(self.shape) - consumed)
            idx = idx[:pos] + fill + idx[pos + 1:]
        return idx

    def __getitem__(self, index):
        return LweSampleArray(
            self.params, self.a[self._a_index(index)], self.b[index], self.current_variances[index])

    def __setitem__(self, index, value):
        if not isinstance(value, LweSampleArray):
            raise ValueError("Only assignment of ciphertexts is supported")
        self.a[self._a_index(index)] = value.a
        self.b[index] = value.b
        self.current_variances[index] = value.current_variances

    def copy(self):
        return LweSampleArray(
            self.params, self.a.clone(), self.b.clone(), self.current_variances.clone())

    def roll(self, shift, axis=-1):
        """In-place cyclic shift along `axis` of the message shape (lwe.py:183-205)."""
        if shift == 0:
            return
        axis = axis % len(self.shape)
        self.a.copy_(torch.roll(self.a, shift, dims=axis))
        self.b.copy_(torch.roll(self.b, shift, dims=axis))
        self.current_variances.copy_(torch.roll(self.current_variances, shift, dims=axis))

    def dump(self, file_obj):
        pickle.dump(self.params, file_obj)
        pickle.dump(self.a.cpu().numpy(), file_obj)
        pickle.dump(self.b.cpu().numpy(), file_obj)
        pickle.dump(self.current_variances.cpu().numpy(), file_obj)

    def dumps(self):
        file_obj = io.BytesIO()
        self.dump(file_obj)
        return file_obj.getvalue()

    @classmethod
    def load(cls, file_obj, thr):
        params = pickle.load(file_obj)
        a = thr.to_device(pickle.load(file_obj))
        b = thr.to_device(pickle.load(file_obj))
        current_variances = thr.to_device(pickle.load(file_obj))
        return cls(params, a, b, current_variances)

    @classmethod
    def loads(cls, s, thr):
        return cls.load(io.BytesIO(s), thr)

    def __eq__(self, other):
        return (self.__class__ == other.__class__ and self.params == other.params
                and arrays_equal(self.a, other.a) and arrays_equal(self.b, other.b)
                and arrays_equal(self.current_variances, other.current_variances))


class LweKeyswitchKey:
    """lwe.py:254-308.  lwe.a: (in, t, base, n) int32, lwe.b / current_variances: (in, t, base)."""

    def __init__(self, lwe: LweSampleArray):
        input_size, decomp_length, base = lwe.shape
        self.lwe = lwe
        self.input_size = input_size
        self.output_size = lwe.params.size
        self.decomp_length = decomp_length
        self.log2_base = int(numpy.log2(base))

    @classmethod
    def from_tgsw_key(cls, thr, rng, ks_decomp_length: int, ks_log2_base: int, lwe_key: LweKey, tgsw_key):
        accum_params = tgsw_key.params.tlwe_params
        extract_params = accum_params.extracted_lweparams
        in_key = LweKey.from_tlwe_key(extract_params, tgsw_key.tlwe_key)
        out_key = lwe_key
        input_size = in_key.params.size
        output_size = out_key.params.size
        noise = out_key.params.min_noise
        base = 2**ks_log2_base

        lwe = LweSampleArray.empty(thr, out_key.params, (input_size, ks_decomp_length, base))
        noises_b = rand_gaussian_torus32(
            thr, rng, 0, noise, (input_size, ks_decomp_length, base - 1), centered=True)
        noises_a = rand_uniform_torus32(
            thr, rng, (input_size, ks_decomp_length, base - 1, output_size))
        make_lwe_keyswitch_key(thr, lwe, in_key.key, out_key.key, noises_a, noises_b, ks_log2_base, noise)
        return cls(lwe)

    def dump(self, file_obj):
        self.lwe.dump(file_obj)

    @classmethod
    def load(cls, file_obj, thr):
        return cls(LweSampleArray.load(file_obj, thr))

    def __eq__(self, other):
        return self.__class__ == other.__class__ and self.lwe == other.lwe

    def device_arrays(self):
        lwe = self.lwe
        return (lwe.a.contiguous(), lwe.b.contiguous(), lwe.current_variances.contiguous())

    def prepare_gemm(self, thr):
        """Register the key for the tensor-core key switch on thr's device (Engine.ks_prepare), once per key array.
        Every key switch with this key's arrays on that engine then uses it, at batches from the library's threshold.
        Engines without it (the CPU test double) and other decomposition parameters keep the gather kernel."""
        prepare = getattr(thr, 'ks_prepare', None)
        if prepare is None or (self.input_size, self.decomp_length, self.log2_base, self.output_size) != (1024, 8, 2, 500):
            return
        if not (self.lwe.a.is_contiguous() and self.lwe.b.is_contiguous()):
            return                              # the registration is for the arrays every key switch passes
        ks_a, ks_b, _ = self.device_arrays()
        cached = getattr(self, '_gemm_planes', None)
        if cached is None or cached[0] is not thr or cached[1] != ks_a.data_ptr():
            self._gemm_planes = (thr, ks_a.data_ptr(), prepare(ks_a, ks_b))


def make_lwe_keyswitch_key(thr, lwe, in_key, out_key, noises_a, noises_b, log2_base, noise):
    """MakeLweKeyswitchKey (lwe_gpu.py:63-124, lwe_gpu.mako:18-56; ref lwe_cpu.py:26-59): row h=0 is
    zero padding, row h encrypts in_key[i] * h * 2^(32 - (j+1) log2_base) under out_key.  One engine kernel
    (nb_make_keyswitch_key); the result arrays of a fresh LweSampleArray are dense."""
    thr.make_keyswitch_key(lwe.a, lwe.b, lwe.current_variances, in_key, out_key, noises_a, noises_b, log2_base,
                           numpy.float32(noise**2))


def _dense_pair(thr, sample: LweSampleArray):
    return (sample.a.contiguous(), sample.b.contiguous())


def lwe_keyswitch(thr, result: LweSampleArray, ks: LweKeyswitchKey, sample: LweSampleArray):
    """lwe.py:311-322 -> K3 (lwe_gpu.mako:59-118)"""
    _keyswitch_into(thr, result, ks, sample, None, 0)


def _keyswitch_into(thr, result, ks, sample1, sample2, const):
    dense = result.a.is_contiguous() and result.b.is_contiguous()
    out = (result.a, result.b) if dense else None
    res_a, res_b, res_cv = thr.keyswitch(
        ks.device_arrays(), _dense_pair(thr, sample1),
        _dense_pair(thr, sample2) if sample2 is not None else None, c=const, out=out, want_cv=True)
    if not dense:
        result.a.copy_(res_a.reshape(result.a.shape))
        result.b.copy_(res_b.reshape(result.b.shape))
    result.current_variances.copy_(res_cv.reshape(result.current_variances.shape))


def lwe_encrypt(thr, rng, result: LweSampleArray, messages, noise: float, key: LweKey):
    """lwe.py:325-333; b = noise + mu + <a, s> (lwe_gpu.py:217-241) -- nb_lwe_dot, no 64-bit temporaries"""
    lwe_size = key.params.size
    noises_b = rand_gaussian_torus32(thr, rng, 0, noise, tuple(messages.shape))
    noises_a = rand_uniform_torus32(thr, rng, tuple(messages.shape) + (lwe_size,))
    result.a.copy_(noises_a)
    b = thr.lwe_dot(noises_a, key.key, add1=messages.to(torch.int32), add2=noises_b, sign=1,
                    out=result.b if result.b.is_contiguous() else None)
    if b is not result.b:
        result.b.copy_(b)
    result.current_variances.fill_(float(numpy.float32(noise**2)))


def lwe_decrypt(thr, sample: LweSampleArray, key: LweKey):
    """lwe.py:336-343; phase = b - <a, s> (lwe_gpu.py:246-284) -- nb_lwe_dot.  Returns a host array."""
    return thr.lwe_dot(sample.a, key.key, add1=sample.b, sign=-1).cpu().numpy()


def _broadcast_source(result_part, source_part, trailing):
    """NumPy-style broadcasting of a source onto the result (lwe_gpu.mako:126-135: size-1 dims index 0)."""
    return source_part.expand(result_part.shape) if source_part.shape != result_part.shape else source_part


def _linear(thr, result: LweSampleArray, source: LweSampleArray, p, add_result):
    """LweLinear (lwe_gpu.py:287-316, lwe_gpu.mako:123-169): result (+)= p * source, with broadcasting."""
    sa = source.a
    sb = source.b
    scv = source.current_variances
    # align leading dims
    nd = result.b.dim()
    while sb.dim() < nd:
        sa, sb, scv = sa.unsqueeze(0), sb.unsqueeze(0), scv.unsqueeze(0)
    sa, sb, scv = sa.expand(result.a.shape), sb.expand(result.b.shape), scv.expand(result.b.shape)
    dense = result.a.is_contiguous() and result.b.is_contiguous()
    if dense:
        x1 = (result.a, result.b) if add_result else None
        thr.lwe_affine((result.a, result.b), x1, (sa.contiguous(), sb.contiguous()), 0, 1, p)
    else:
        pa = (sa.to(torch.int64) * p + (result.a.to(torch.int64) if add_result else 0)) & 0xffffffff
        pb = (sb.to(torch.int64) * p + (result.b.to(torch.int64) if add_result else 0)) & 0xffffffff
        result.a.copy_(torch.where(pa >= 2**31, pa - 2**32, pa).to(torch.int32))
        result.b.copy_(torch.where(pb >= 2**31, pb - 2**32, pb).to(torch.int32))
    cv = scv * float(p * p)
    result.current_variances.copy_(result.current_variances + cv if add_result else cv)


def lwe_noiseless_trivial(thr, result: LweSampleArray, mus):
    """lwe.py:346-351: (0, mu) for each mu (broadcast onto result)"""
    result.a.zero_()
    result.b.copy_(mus.expand(result.b.shape) if tuple(mus.shape) != tuple(result.b.shape) else mus)
    result.current_variances.zero_()


def lwe_noiseless_trivial_constant(thr, result: LweSampleArray, mu):
    """lwe.py:354-359"""
    result.a.zero_()
    result.b.fill_(int(mu))
    result.current_variances.zero_()


def lwe_negate(thr, result, source):
    _linear(thr, result, source, -1, False)


def lwe_copy(thr, result, source):
    _linear(thr, result, source, 1, False)


def lwe_add_to(thr, result, source):
    _linear(thr, result, source, 1, True)


def lwe_add_mul_to(thr, result, p: int, source):
    _linear(thr, result, source, p, True)


def lwe_sub_to(thr, result, source):
    _linear(thr, result, source, -1, True)


def lwe_sub_mul_to(thr, result, p: int, source):
    _linear(thr, result, source, -p, True)


def concatenate(lwe_sample_arrays, axis=0, out=None):
    """lwe.py:425-447"""
    if len(lwe_sample_arrays) == 0:
        raise ValueError("Need at least one ciphertext to concatenate")
    params = lwe_sample_arrays[0].params
    nd = len(lwe_sample_arrays[0].shape)
    axis = axis % nd
    lwes_a = [lwe.a for lwe in lwe_sample_arrays]
    lwes_b = [lwe.b for lwe in lwe_sample_arrays]
    lwes_cv = [lwe.current_variances for lwe in lwe_sample_arrays]
    if out is None:
        out = LweSampleArray(
            params, torch.cat(lwes_a, dim=axis), torch.cat(lwes_b, dim=axis), torch.cat(lwes_cv, dim=axis))
    else:
        out.a.copy_(torch.cat(lwes_a, dim=axis))
        out.b.copy_(torch.cat(lwes_b, dim=axis))
        out.current_variances.copy_(torch.cat(lwes_cv, dim=axis))
    return out
