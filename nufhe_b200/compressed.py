"""Compressed cloud keys and ciphertexts (DESIGN.md section 10).

The uniform masks of LWE / TLWE samples carry no information, so a compressed object stores a 256-bit seed instead and
the engine regenerates the masks from it with ChaCha20 (Engine.seeded_uniform, nb_seeded_uniform_i32).  Streams:

    object               seed                       nonce   mask layout (C order)
    ciphertext array     its own, per encryption    0       shape + (n,)
    bootstrap key        the cloud key's seed       1       (n, k+1, l, k, N): the TLWE masks, polys [..., :k, :]
    key-switch key       the cloud key's seed       2       (in, t, base-1, n_out); rows h = 0 stay zero
    packing key          its own                    4       (n, t, k, N)
    tree key             its own                    5       (n, t, k, N)
    encrypted index      its own, per encryption    6       (rows, k+1, l, k, N), rows = shape x bits (index_lookup.py)
    compact public key   its own                    7       (k, N) (compact.py)
    compact encryption   its own, per encryption    8       (G, N / 32) words of the binary polynomials r (compact.py)

Seeds are drawn from the context RNG as `rng.uniform_torus32((8,))`.  `decompress()` gives the ordinary objects
(LweSampleArray, NuFHECloudKey) that the rest of the library takes.

The bootstrap key cannot take the usual `tgsw_add_message`, which adds m * h_j to coefficient 0 of mask polynomial mi
for rows mi < k: a seeded mask cannot carry it, and storing the corrected coefficient would publish m, a bit of the
secret LWE key.  The rows mi < k get the phase-equivalent body instead, body = e + sum_u a_u S_u - m h_j S_mi, so that
body - sum_u a_u S_u equals the phase of an ordinary TGSW row; the external product depends on the phases only."""
import io
import pickle

import numpy
import torch

from .lwe import LweParams, LweSampleArray, LweKey, LweKeyswitchKey, make_lwe_keyswitch_key
from .tlwe import tlwe_encrypt_zero_with_masks
from .tgsw import TGswKey, TGswSampleArray, TransformedTGswSampleArray, tgsw_transform_samples
from .bootstrap import BootstrapKey, MultiBitBootstrapKey, MultiBitTGswSampleArray, check_multi_bit, multi_bit_messages
from .random_numbers import rand_gaussian_torus32

NONCE_CIPHERTEXT, NONCE_BOOTSTRAP_KEY, NONCE_KEYSWITCH_KEY = 0, 1, 2

_CIPHERTEXT_TAG = 'nufhe_b200.CompressedLweSampleArray/1'
_CLOUD_KEY_TAG = 'nufhe_b200.CompressedCloudKey/1'


def draw_seed(rng):
    """A 256-bit seed: 8 Torus32 draws of the context RNG (32 bytes of os.urandom for SecureRNG), as uint32."""
    return numpy.asarray(rng.uniform_torus32((8,))).astype(numpy.int32).view(numpy.uint32).copy()


def _check_tag(file_obj, tag):
    try:
        got = pickle.load(file_obj)
    except Exception as e:
        raise ValueError('not a %s pickle: %s' % (tag.split('/')[0], e)) from e
    if not isinstance(got, str) or got != tag:
        raise ValueError('not a %s pickle (format tag %r)' % (tag.split('/')[0], got if isinstance(got, str) else type(got).__name__))


def _variance(noise):
    """The variance a fresh sample records (lwe_encrypt, tlwe_encrypt_zero)."""
    return float(numpy.float32(noise**2))


class CompressedLweSampleArray:
    """An encrypted array without its masks: params, message shape, seed, body `b` (shape) int32 and the one variance
    every fresh sample has.  `decompress(thr)` gives the LweSampleArray."""

    def __init__(self, params: LweParams, shape, seed, b, variance: float):
        self.params = params
        self.shape = tuple(shape)
        self.seed = numpy.asarray(seed, numpy.uint32).reshape(8)
        self.b = b
        self.variance = float(variance)
        if tuple(b.shape) != self.shape:
            raise ValueError('body shape %s does not match %s' % (tuple(b.shape), self.shape))

    @classmethod
    def encrypt(cls, thr, rng, params: LweParams, mus, noise: float, key: LweKey):
        """lwe_encrypt with the mask from a fresh seed: draws the seed, then the Gaussian noises of b in lwe_encrypt's
        order; b = mu + e + <a, s> (nb_lwe_dot)."""
        shape = tuple(mus.shape)
        seed = draw_seed(rng)
        noises_b = rand_gaussian_torus32(thr, rng, 0, noise, shape)
        a = thr.seeded_uniform(seed, NONCE_CIPHERTEXT, shape + (params.size,))
        b = thr.lwe_dot(a, key.key, add1=mus.to(torch.int32), add2=noises_b, sign=1)
        return cls(params, shape, seed, b, _variance(noise))

    def decompress(self, thr):
        a = thr.seeded_uniform(self.seed, NONCE_CIPHERTEXT, self.shape + (self.params.size,))
        b = self.b.to(thr.device).clone()
        cv = torch.empty(self.shape, dtype=torch.float32, device=b.device)
        cv.fill_(self.variance)
        return LweSampleArray(self.params, a, b, cv)

    def dump(self, file_obj):
        pickle.dump(_CIPHERTEXT_TAG, file_obj)
        pickle.dump(self.params, file_obj)
        pickle.dump(self.shape, file_obj)
        pickle.dump(self.seed, file_obj)
        pickle.dump(self.b.cpu().numpy(), file_obj)
        pickle.dump(self.variance, file_obj)

    def dumps(self):
        file_obj = io.BytesIO()
        self.dump(file_obj)
        return file_obj.getvalue()

    @classmethod
    def load(cls, file_obj, thr):
        _check_tag(file_obj, _CIPHERTEXT_TAG)
        params = pickle.load(file_obj)
        shape = pickle.load(file_obj)
        seed = pickle.load(file_obj)
        b = thr.to_device(pickle.load(file_obj)).reshape(shape)     # (to_device makes a scalar 1-D)
        variance = pickle.load(file_obj)
        return cls(params, shape, seed, b, variance)

    @classmethod
    def loads(cls, s: bytes, thr):
        return cls.load(io.BytesIO(s), thr)

    def __eq__(self, other):
        return (self.__class__ == other.__class__ and self.params == other.params and self.shape == other.shape
                and (self.seed == other.seed).all() and torch.equal(self.b.cpu(), other.b.cpu())
                and self.variance == other.variance)


def _bk_masks(thr, seed, params, n):
    k, l, N = params.tlwe_params.mask_size, params.decomp_length, params.tlwe_params.polynomial_degree
    return thr.seeded_uniform(seed, NONCE_BOOTSTRAP_KEY, (n, k + 1, l, k, N))


def _ks_masks(thr, seed, in_size, t, base, n_out):
    return thr.seeded_uniform(seed, NONCE_KEYSWITCH_KEY, (in_size, t, base - 1, n_out))


def _wrap32(x):
    return torch.where(x >= 2**31, x - 2**32, x).to(torch.int32)


def tgsw_add_message_seeded(thr, result: TGswSampleArray, messages, key: TGswKey):
    """The phase of result += m * H without touching the masks: row mi < k, level j gets -m h_j S_mi on its body,
    row mi = k gets m h_j on coefficient 0 of its body (tgsw_add_message adds the same phases through the masks)."""
    params = result.params
    k = params.tlwe_params.mask_size
    coeffs = result.samples.a.coeffs                                   # (n, k+1, l, k+1, N)
    h = torch.from_numpy(params.base_powers.astype(numpy.int64)).to(coeffs.device)
    inc = messages.to(torch.int64).reshape(-1, 1) * h.reshape(1, -1)  # (n, l): m h_j
    s = key.tlwe_key.key.coeffs.to(torch.int64)                        # (k, N)
    for mi in range(k):
        v = (coeffs[:, mi, :, k, :].to(torch.int64) - inc[:, :, None] * s[mi][None, None, :]) & 0xffffffff
        coeffs[:, mi, :, k, :] = _wrap32(v)
    v = (coeffs[:, k, :, k, 0].to(torch.int64) + inc) & 0xffffffff
    coeffs[:, k, :, k, 0] = _wrap32(v)


class CompressedCloudKey:
    """A cloud key whose masks are regenerated from one seed: the bootstrap key's TLWE bodies (n, k+1, l, N) int32 and
    their variance, the key-switch key's bodies (in, t, base) int32 and its variance.  About 8.3 MB for the default
    parameters, against 98.6 MB for the NuFHECloudKey that `decompress(thr)` rebuilds."""

    def __init__(self, params, seed, bk_body, bk_variance, ks_b, ks_variance):
        self.params = params
        self.seed = numpy.asarray(seed, numpy.uint32).reshape(8)
        self.bk_body = bk_body
        self.bk_variance = float(bk_variance)
        self.ks_b = ks_b
        self.ks_variance = float(ks_variance)

    @classmethod
    def from_rng(cls, thr, params, rng, secret_key):
        """Key generation in the order: TGSW key, seed, bootstrap-key body noises, key-switch noises_b."""
        return cls.from_rng_with_tgsw_key(thr, params, rng, secret_key)[0]

    @classmethod
    def from_rng_with_tgsw_key(cls, thr, params, rng, secret_key, multi_bit=1):
        """(compressed cloud key, TGswKey), as NuFHECloudKey.from_rng_with_tgsw_key.  multi_bit=2: the 3n/2 rows of a
        MultiBitBootstrapKey take the bootstrap key's place (bodies, masks and draws), which `decompress` restores."""
        check_multi_bit(params, multi_bit)
        lwe_key = secret_key.lwe_key
        tgsw_key = TGswKey.from_rng(thr, params.tgsw_params, rng)
        seed = draw_seed(rng)
        bk_params = params.tgsw_params
        tl = bk_params.tlwe_params
        n = lwe_key.params.size
        rows, messages = (3 * n // 2, multi_bit_messages(lwe_key.key)) if multi_bit == 2 else (n, lwe_key.key)

        bk = TGswSampleArray.empty(thr, bk_params, (rows,))
        noises2 = rand_gaussian_torus32(thr, rng, 0, tl.min_noise, bk.samples.shape + (tl.polynomial_degree,))
        tlwe_encrypt_zero_with_masks(thr, bk.samples, _bk_masks(thr, seed, bk_params, rows), noises2, tl.min_noise,
                                     tgsw_key.tlwe_key)
        tgsw_add_message_seeded(thr, bk, messages, tgsw_key)
        k = tl.mask_size
        bk_body = bk.samples.a.coeffs[..., k, :].contiguous()

        in_key = LweKey.from_tlwe_key(tl.extracted_lweparams, tgsw_key.tlwe_key)
        t, base = params.ks_decomp_length, 2**params.ks_log2_base
        in_size, n_out = in_key.params.size, lwe_key.params.size
        noise = lwe_key.params.min_noise
        noises_b = rand_gaussian_torus32(thr, rng, 0, noise, (in_size, t, base - 1), centered=True)
        ks = LweSampleArray.empty(thr, lwe_key.params, (in_size, t, base))
        make_lwe_keyswitch_key(thr, ks, in_key.key, lwe_key.key, _ks_masks(thr, seed, in_size, t, base, n_out),
                               noises_b, params.ks_log2_base, noise)
        return cls(params, seed, bk_body, _variance(tl.min_noise), ks.b.contiguous(), _variance(noise)), tgsw_key

    def decompress(self, thr):
        """The NuFHECloudKey: masks regenerated on the device, the bootstrap key transformed as at key generation."""
        from .api_low_level import NuFHECloudKey
        params = self.params
        bk_params = params.tgsw_params
        k = bk_params.tlwe_params.mask_size
        n = params.in_out_params.size
        rows = self.bk_body.shape[0]                 # n, or 3n/2 for a multi-bit key
        bk = TGswSampleArray.empty(thr, bk_params, (rows,))
        coeffs = bk.samples.a.coeffs
        coeffs[..., :k, :] = _bk_masks(thr, self.seed, bk_params, rows)
        coeffs[..., k, :] = self.bk_body.to(coeffs.device)
        bk.samples.current_variances.fill_(self.bk_variance)
        multi = rows != n
        bk_transformed = (MultiBitTGswSampleArray if multi else TransformedTGswSampleArray).empty(thr, bk_params, (rows,))
        tgsw_transform_samples(thr, bk_transformed, bk)
        bootstrap_key = (MultiBitBootstrapKey if multi else BootstrapKey)(params.in_out_params, bk_transformed)

        in_size, t, base = self.ks_b.shape
        ks = LweSampleArray.empty(thr, params.in_out_params, (in_size, t, base))
        ks.a[:, :, 0, :] = 0
        ks.a[:, :, 1:, :] = _ks_masks(thr, self.seed, in_size, t, base, n)
        ks.b.copy_(self.ks_b.to(ks.b.device))
        ks.current_variances.zero_()
        ks.current_variances[:, :, 1:] = self.ks_variance
        return NuFHECloudKey(params, bootstrap_key, LweKeyswitchKey(ks))

    def dump(self, file_obj):
        pickle.dump(_CLOUD_KEY_TAG, file_obj)
        pickle.dump(self.params, file_obj)
        pickle.dump(self.seed, file_obj)
        pickle.dump(self.bk_body.cpu().numpy(), file_obj)
        pickle.dump(self.bk_variance, file_obj)
        pickle.dump(self.ks_b.cpu().numpy(), file_obj)
        pickle.dump(self.ks_variance, file_obj)

    def dumps(self):
        file_obj = io.BytesIO()
        self.dump(file_obj)
        return file_obj.getvalue()

    @classmethod
    def load(cls, file_obj, thr):
        _check_tag(file_obj, _CLOUD_KEY_TAG)
        params = pickle.load(file_obj)
        seed = pickle.load(file_obj)
        bk_body = thr.to_device(pickle.load(file_obj))
        bk_variance = pickle.load(file_obj)
        ks_b = thr.to_device(pickle.load(file_obj))
        ks_variance = pickle.load(file_obj)
        return cls(params, seed, bk_body, bk_variance, ks_b, ks_variance)

    @classmethod
    def loads(cls, s: bytes, thr):
        return cls.load(io.BytesIO(s), thr)

    def __eq__(self, other):
        return (self.__class__ == other.__class__ and self.params == other.params and (self.seed == other.seed).all()
                and torch.equal(self.bk_body.cpu(), other.bk_body.cpu()) and self.bk_variance == other.bk_variance
                and torch.equal(self.ks_b.cpu(), other.ks_b.cpu()) and self.ks_variance == other.ks_variance)
