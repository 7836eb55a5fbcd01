"""Public-key encryption (DESIGN.md section 11).

A public key is m LWE encryptions of 0 under the secret LWE key, stored compressed: the seed of its masks A (m, n)
(ChaCha20 stream (seed, nonce 0), as for any compressed ciphertext) and its bodies b (m,).  Anyone holding it encrypts
B messages as

    (a, b) = R [A | b_pk] + (0, mu)        R a fresh secret uniform binary (B, m) matrix,

one integer GEMM on the tensor cores (nb_pk_encrypt).  R is expanded from a seed drawn per call and never stored:
stream (r_seed, nonce 3) as (B, m/32) words, bit i of row c = bit i % 32 of word (c, i // 32)."""
import io
import pickle

import numpy
import torch

from .lwe import LweSampleArray
from .compressed import CompressedLweSampleArray, NONCE_CIPHERTEXT, draw_seed, _check_tag

NONCE_ENCRYPTION_RANDOMNESS = 3

_PUBLIC_KEY_TAG = 'nufhe_b200.NuFHEPublicKey/1'


def public_key_size(params):
    """m, the number of encryptions of 0 in a public key: m >= (n + 1) * 32 + 256 rounded up to a multiple of 1024
    (16 384 for n = 500), enough for the leftover hash lemma with a binary R."""
    n = params.in_out_params.size
    return 1024 * (((n + 1) * 32 + 256 + 1023) // 1024)


class NuFHEPublicKey:
    """params, the 256-bit seed of the masks, the bodies `b` (m,) int32 and the variance of each row's noise.  About
    66 KB pickled for the default parameters.  `ctx.encrypt(pk, bits)` and `ctx.encrypt_int(pk, values, bits)` take it
    in place of the secret key."""

    def __init__(self, params, seed, b, variance: float):
        self.params = params
        self.seed = numpy.asarray(seed, numpy.uint32).reshape(8)
        self.b = b
        self.variance = float(variance)
        if tuple(b.shape) != (public_key_size(params),):
            raise ValueError('a public key for these parameters has %d rows, got body shape %s'
                             % (public_key_size(params), tuple(b.shape)))
        self._planes = None

    @classmethod
    def from_secret_key(cls, thr, rng, secret_key):
        """A compressed encryption of m zeros with the fresh-encryption noise: draws the seed, then m Gaussians."""
        params = secret_key.params
        io_params = params.in_out_params
        zeros = thr.to_device(numpy.zeros(public_key_size(params), numpy.int32))
        ct = CompressedLweSampleArray.encrypt(thr, rng, io_params, zeros, io_params.min_noise, secret_key.lwe_key)
        return cls(params, ct.seed, ct.b, ct.variance)

    @property
    def size(self):
        return int(self.b.shape[0])

    def masks(self, thr):
        """The masks A (m, n), regenerated from the seed."""
        return thr.seeded_uniform(self.seed, NONCE_CIPHERTEXT, (self.size, self.params.in_out_params.size))

    def planes(self, thr):
        """[A | b | 1] in the byte planes nb_pk_encrypt reads (nb_pk_prepare), built once per engine and cached."""
        if self._planes is None or self._planes[0] is not thr:
            self._planes = (thr, thr.pk_prepare(self.masks(thr), self.b.to(thr.device)))
        return self._planes[1]

    def dump(self, file_obj):
        pickle.dump(_PUBLIC_KEY_TAG, file_obj)
        pickle.dump(self.params, file_obj)
        pickle.dump(self.seed, file_obj)
        pickle.dump(self.b.cpu().numpy(), file_obj)
        pickle.dump(self.variance, file_obj)

    def dumps(self):
        file_obj = io.BytesIO()
        self.dump(file_obj)
        return file_obj.getvalue()

    @classmethod
    def load(cls, file_obj, thr):
        _check_tag(file_obj, _PUBLIC_KEY_TAG)
        params = pickle.load(file_obj)
        seed = pickle.load(file_obj)
        b = thr.to_device(pickle.load(file_obj))
        variance = pickle.load(file_obj)
        return cls(params, seed, b, variance)

    @classmethod
    def loads(cls, s: bytes, thr):
        return cls.load(io.BytesIO(s), thr)

    def __eq__(self, other):
        return (self.__class__ == other.__class__ and self.params == other.params and (self.seed == other.seed).all()
                and torch.equal(self.b.cpu(), other.b.cpu()) and self.variance == other.variance)


def public_encrypt(thr, rng, pk: NuFHEPublicKey, mus):
    """Encrypt the Torus32 messages `mus` (a device int32 tensor of any shape) with the public key.  Draws one 256-bit
    seed from `rng` and nothing else; the ciphertexts' variances are popcount(r_c) times the key's row variance."""
    shape = tuple(mus.shape)
    io_params = pk.params.in_out_params
    m, n = pk.size, io_params.size
    r_seed = draw_seed(rng)
    batch = int(numpy.prod(shape, dtype=numpy.int64))
    r_words = thr.seeded_uniform(r_seed, NONCE_ENCRYPTION_RANDOMNESS, (batch, m // 32))
    a, b, cv = thr.public_encrypt(r_words, pk.planes(thr), m, n, mus.reshape(-1), pk.variance)
    return LweSampleArray(io_params, a.reshape(shape + (n,)), b.reshape(shape), cv.reshape(shape))
