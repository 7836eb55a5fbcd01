"""Bootstrap key and the bootstrap procedure (reference: nufhe/bootstrap.py)."""
import pickle

import torch

from .numeric_functions import Torus32, t32_to_phase
from .lwe import LweParams, LweKey, LweSampleArray, LweKeyswitchKey, _keyswitch_into, lwe_keyswitch
from .polynomials import TorusPolynomialArray, shift_tp_inverted_power
from .tlwe import (
    TLweSampleArray, tlwe_noiseless_trivial, tlwe_extract_lwe_samples, tlwe_shift_polynomials, tlwe_add_to, tlwe_copy)
from .tgsw import (
    TGswKey, TransformedTGswSampleArray, TGswParams, TGswSampleArray,
    tgsw_transform_samples, tgsw_encrypt_int, tgsw_transformed_external_mul, engine_format, fused_kernel_supported)


class BootstrapKey:
    """bootstrap.py:44-92"""

    def __init__(self, in_out_params: LweParams, tgsw: TransformedTGswSampleArray):
        bk_params = tgsw.params
        accum_params = bk_params.tlwe_params
        self.in_out_params = in_out_params
        self.bk_params = bk_params
        self.accum_params = accum_params
        self.extract_params = accum_params.extracted_lweparams
        self.tgsw = tgsw

    @classmethod
    def from_rng(cls, thr, rng, lwe_key: LweKey, tgsw_key: TGswKey, perf_params=None):
        in_out_params = lwe_key.params
        bk_params = tgsw_key.params
        accum_params = bk_params.tlwe_params
        bk = TGswSampleArray.empty(thr, bk_params, (in_out_params.size,))
        tgsw_encrypt_int(thr, rng, bk, lwe_key.key, accum_params.min_noise, tgsw_key, perf_params)
        bk_transformed = TransformedTGswSampleArray.empty(thr, bk_params, (in_out_params.size,))
        tgsw_transform_samples(thr, bk_transformed, bk, perf_params)
        return cls(in_out_params, bk_transformed)

    def dump(self, file_obj):
        pickle.dump(self.in_out_params, file_obj)
        self.tgsw.dump(file_obj)

    @classmethod
    def load(cls, file_obj, thr):
        """A BootstrapKey, or the MultiBitBootstrapKey whose pickle starts with its tag."""
        in_out_params = pickle.load(file_obj)
        if isinstance(in_out_params, str):
            if in_out_params != MULTI_BIT_TAG:
                raise ValueError('not a bootstrap key: %r' % in_out_params)
            in_out_params = pickle.load(file_obj)
            return MultiBitBootstrapKey(in_out_params, MultiBitTGswSampleArray.load(file_obj, thr))
        tgsw = TransformedTGswSampleArray.load(file_obj, thr)
        return cls(in_out_params, tgsw)

    def __eq__(self, other):
        return (self.__class__ == other.__class__ and self.in_out_params == other.in_out_params
                and self.tgsw == other.tgsw)


MULTI_BIT_TAG = 'nufhe_b200.MultiBitBootstrapKey/1'


def check_multi_bit(params, multi_bit):
    """Raise for a `multi_bit` choice the key's parameters cannot take (`params`: NuFHEParameters)."""
    if isinstance(multi_bit, bool) or not isinstance(multi_bit, int):
        raise TypeError('multi_bit must be the integer 1 or 2, got %r' % (multi_bit,))
    if multi_bit not in (1, 2):
        raise ValueError('multi_bit must be 1 (one key bit per CMux step) or 2 (two), got %d' % multi_bit)
    if multi_bit == 1:
        return
    if params.tgsw_params.tlwe_params.mask_size != 1 or not fused_kernel_supported(params.tgsw_params):
        raise ValueError('multi-bit bootstrap keys run on the fused kernel only: tlwe_mask_size = 1, the default '
                         'decomposition and N = 1024')
    if params.in_out_params.size % 2:
        raise ValueError('a multi-bit bootstrap key takes the key bits in pairs: the LWE dimension must be even, '
                         'got %d' % params.in_out_params.size)


def multi_bit_messages(key_bits):
    """The (3n/2,) indicators a multi-bit key encrypts: row 3 g + p - 1 holds [s_2g = b0 and s_2g+1 = b1], p = b0 + 2 b1."""
    s = key_bits.to(torch.int32).reshape(-1, 2)
    s0, s1 = s[:, 0], s[:, 1]
    return torch.stack([s0 * (1 - s1), (1 - s0) * s1, s0 * s1], dim=1).reshape(-1).contiguous()


class MultiBitTGswSampleArray(TransformedTGswSampleArray):
    """The rows of a multi-bit bootstrap key, (3n/2, k+1, l, k+1, N) in the reference's transformed wire format.
    engine_format lays them out for the multi-bit kernels (nb_bk_prepare_multibit)."""
    multi_bit = 2


class MultiBitBootstrapKey(BootstrapKey):
    """A bootstrap key that takes the key bits two at a time (DESIGN.md section 14): 3n/2 TGSW rows, row 3 g + p - 1
    encrypting the indicator [s_2g = b0 and s_2g+1 = b1] of pattern p = b0 + 2 b1 = 1, 2, 3.  The blind rotation runs
    n/2 steps of ACC += sum_p (X^{k_p} - 1) (Dec(ACC) [x] BK_{g,p}).  Gates, lookup tables and lut_tree take it as they
    take a BootstrapKey; the separate-step bootstrap (single_kernel_bootstrap=False) and blind_rotate do not."""
    multi_bit = 2

    @classmethod
    def from_rng(cls, thr, rng, lwe_key: LweKey, tgsw_key: TGswKey, perf_params=None):
        """The rows are drawn where a BootstrapKey's are, 3n/2 TGSW encryptions in row order."""
        in_out_params = lwe_key.params
        bk_params = tgsw_key.params
        accum_params = bk_params.tlwe_params
        rows = 3 * in_out_params.size // 2
        bk = TGswSampleArray.empty(thr, bk_params, (rows,))
        tgsw_encrypt_int(thr, rng, bk, multi_bit_messages(lwe_key.key), accum_params.min_noise, tgsw_key, perf_params)
        bk_transformed = MultiBitTGswSampleArray.empty(thr, bk_params, (rows,))
        tgsw_transform_samples(thr, bk_transformed, bk, perf_params)
        return cls(in_out_params, bk_transformed)

    def dump(self, file_obj):
        pickle.dump(MULTI_BIT_TAG, file_obj)
        BootstrapKey.dump(self, file_obj)


def _flat(sample: LweSampleArray):
    return (sample.a.contiguous(), sample.b.contiguous())


def bootstrap_affine(thr, result: LweSampleArray, bk: BootstrapKey, ks: LweKeyswitchKey, mu,
                     x1: LweSampleArray, x2, c, s1, s2, no_keyswitch=False):
    """bootstrap(mu, (0,c) + s1*x1 + s2*x2): the gates' linear prologue (gates.py:108-115), the
    mod-switch, test-vector rotation, 500-step blind rotation and sample extraction run as ONE kernel
    (nb_bootstrap_extract), followed by the key-switch kernel unless `no_keyswitch`."""
    bk_int = engine_format(thr, bk.tgsw)
    shape = tuple(result.shape)

    def expand(x):
        if x is None:
            return None
        a, b = x.a, x.b
        if tuple(b.shape) != shape:
            while b.dim() < len(shape):
                a, b = a.unsqueeze(0), b.unsqueeze(0)
            a, b = a.expand(shape + (a.shape[-1],)), b.expand(shape)
        return (a.contiguous(), b.contiguous())

    p1, p2 = expand(x1), expand(x2)
    if no_keyswitch:
        dense = result.a.is_contiguous() and result.b.is_contiguous()
        out = (result.a, result.b) if dense else None
        ext = thr.bootstrap_extract(p1, p2, c, s1, s2, mu, bk_int, out=out)
        if not dense:
            result.a.copy_(ext[0].reshape(result.a.shape))
            result.b.copy_(ext[1].reshape(result.b.shape))
        result.current_variances.zero_()
    else:
        ext = thr.bootstrap_extract(p1, p2, c, s1, s2, mu, bk_int)
        ext_sample = LweSampleArray(
            bk.extract_params, ext[0].reshape(shape + (ext[0].shape[-1],)), ext[1].reshape(shape),
            torch.zeros(shape, dtype=torch.float32, device=ext[1].device))
        _keyswitch_into(thr, result, ks, ext_sample, None, 0)


def _single_kernel(perf_params, bk=None):
    """Which bootstrap path to take.  Without explicit performance parameters: the fused kernel whenever the key's
    parameters allow it (what `PerformanceParameters(params).for_device(...)` would say)."""
    if getattr(bk, 'multi_bit', 1) == 2:
        if perf_params is not None and getattr(perf_params, 'single_kernel_bootstrap', True) is False:
            raise ValueError('a multi-bit bootstrap key runs on the fused kernel only (single_kernel_bootstrap=True)')
        return True
    if perf_params is None:
        return bk is None or fused_kernel_supported(bk.bk_params)
    return getattr(perf_params, 'single_kernel_bootstrap', True) is not False


def mux_rotate(thr, result: TLweSampleArray, accum: TLweSampleArray, bki: TransformedTGswSampleArray, bk_idx: int,
               barai, bk_params: TGswParams = None, perf_params=None):
    """result = BK_i (x) ((X^barai - 1) accum) + accum  (bootstrap.py:96-109): three launches."""
    tlwe_shift_polynomials(thr, result, accum, barai, bk_idx)
    tgsw_transformed_external_mul(thr, result, bki, bk_idx, perf_params)
    tlwe_add_to(thr, result, accum)


def blind_rotate(thr, accum: TLweSampleArray, bk: BootstrapKey, bara, n: int, bk_params: TGswParams = None,
                 perf_params=None):
    """accum <- X^(sum_i bara_i s_i) * accum, one CMux per key row with two ping-pong buffers (bootstrap.py:120-142)."""
    temp = TLweSampleArray.empty(thr, bk.bk_params.tlwe_params, accum.shape)
    temp2, temp3 = temp, accum
    accum_in_temp3 = True
    for i in range(n):
        mux_rotate(thr, temp2, temp3, bk.tgsw, i, bara, bk_params, perf_params)
        temp2, temp3 = temp3, temp2
        accum_in_temp3 = not accum_in_temp3
    if not accum_in_temp3:
        tlwe_copy(thr, accum, temp3)


def blind_rotate_and_extract(thr, result: LweSampleArray, v: TorusPolynomialArray, bk: BootstrapKey,
                             ks: LweKeyswitchKey, barb, bara, perf_params=None, no_keyswitch=False):
    """result = LWE(v_p), p = barb - sum bara_i s_i mod 2N (bootstrap.py:154-196).  With
    `perf_params.single_kernel_bootstrap` false the rotation is the literal loop of separate launches."""
    from .blind_rotate import BlindRotate_gpu
    accum_params = bk.bk_params.tlwe_params
    shape = tuple(result.shape)
    extracted = result if no_keyswitch else LweSampleArray.empty(thr, bk.extract_params, shape)
    testvectbis = TorusPolynomialArray.empty(thr, accum_params.polynomial_degree, shape)
    shift_tp_inverted_power(thr, testvectbis, barb, v)
    acc = TLweSampleArray.empty(thr, accum_params, shape)
    tlwe_noiseless_trivial(thr, acc, testvectbis)
    if _single_kernel(perf_params, bk):
        BlindRotate_gpu(result, acc, bk, ks, bara, perf_params, no_keyswitch=no_keyswitch, thr=thr)
    else:
        blind_rotate(thr, acc, bk, bara, bk.in_out_params.size, bk.bk_params, perf_params)
        tlwe_extract_lwe_samples(thr, extracted, acc)
        if not no_keyswitch:
            lwe_keyswitch(thr, result, ks, extracted)


def bootstrap(thr, result: LweSampleArray, bk: BootstrapKey, ks: LweKeyswitchKey, mu,
              x: LweSampleArray, perf_params=None, no_keyswitch=False):
    """bootstrap.py:206-229: result = LWE(mu) iff phase(x) > 0, LWE(-mu) otherwise.
    Default: one fused kernel (+ key switch).  `single_kernel_bootstrap=False`: the reference's sequence of
    separate steps -- mod-switch, test vector, rotation of the test vector, trivial sample, 500 x 3 launches,
    extraction, key switch -- with bit-identical results (tests/test_gpu_api.py)."""
    if _single_kernel(perf_params, bk):
        bootstrap_affine(thr, result, bk, ks, mu, x, None, 0, 1, 0, no_keyswitch=no_keyswitch)
        return
    N = bk.accum_params.polynomial_degree
    xa, xb = x.a.contiguous(), x.b.contiguous()
    barb = torch.empty(tuple(xb.shape), dtype=torch.int32, device=xb.device)
    bara = torch.empty(tuple(xa.shape), dtype=torch.int32, device=xa.device)
    t32_to_phase(thr, barb, xb, 2 * N)
    t32_to_phase(thr, bara, xa, 2 * N)
    testvect = TorusPolynomialArray.empty(thr, N, tuple(result.shape))
    testvect.coeffs.fill_(int(mu))
    blind_rotate_and_extract(thr, result, testvect, bk, ks, barb, bara, perf_params, no_keyswitch=no_keyswitch)
