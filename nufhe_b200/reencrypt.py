"""Re-encryption (DESIGN.md section 22): move LWE ciphertexts from one client's key to another's on the server, without
decrypting them and without the recipient's secret.

A re-encryption key from client A to client B is one GLWE sample C = (A_C, B_C) under B's bootstrap-key GLWE key S_B,
made by A from B's compact public key (section 16) as compact_encrypt makes one group, but without the 16-bit rounding:
slot p = 2 i + j holds s_A[i] g_j (g_0 = 2^24, g_1 = 2^16, packing's gadget), slots 2 n .. N - 1 hold 0.  8 KB for k = 1.

Re-encrypting (a, b) under s_A: with the signed 8-bit digits d_p = d_j(a_i) (pack_digit), (0, b) - sum_p d_p
extract_p(C) is an LWE sample under the extracted key of S_B whose phase is b - sum_i s_A[i] round_16(a_i); its mask is
one exact negacyclic product D . A_C and its body a dot product with B_C (nb_reencrypt).  B's cloud-key key switch then
takes it to s_B."""
import io
import pickle

import numpy
import torch

from .lwe import LweSampleArray
from .compact import NuFHECompactPublicKey, noise_terms, r_bits, _fields, _glwe, PASS_BYTES
from .compressed import draw_seed, _check_tag
from .random_numbers import rand_gaussian_torus32
from .batch_keys import OneKey, owners
from . import lut, index_lookup

LEVELS = 2                                # t: digits per mask word
GADGET = (1 << 24, 1 << 16)               # g_0, g_1
DIGIT_SQUARE = sum(d * d for d in range(-128, 128)) / 256      # E[d^2] of a uniform signed 8-bit digit: 5461.5

_KEY_TAG = 'nufhe_b200.NuFHEReencryptionKey/1'


def _check_shape(params, n):
    tl, k, N = _glwe(params)
    if k != 1 or LEVELS * n > N:
        raise ValueError('re-encryption keys are for k = 1 and n t <= N only (k = %d, n = %d)' % (k, n))


class NuFHEReencryptionKey:
    """params, n (the LWE dimension of the sender's key) and `sample` (k + 1, N) int32: one GLWE sample under the
    recipient's S_B whose slot 2 i + j encrypts s_A[i] g_j.  8 KB of data for k = 1.  `spectra(thr)` -- the NTT of the
    mask and the body, what nb_reencrypt reads -- is built once per engine and cached on the object."""

    def __init__(self, params, n, sample):
        self.params = params
        self.n = int(n)
        self.sample = sample
        tl, k, N = _glwe(params)
        _check_shape(params, self.n)
        if tuple(sample.shape) != (k + 1, N) or sample.dtype != torch.int32:
            raise ValueError('a re-encryption key for these parameters is int32 %s, got %s %s'
                             % ((k + 1, N), sample.dtype, tuple(sample.shape)))
        self._spectra = None

    def spectra(self, thr):
        """(mask spectrum (k, N) field elements, body (N,) int32) on the engine's device."""
        if self._spectra is None or self._spectra[0] is not thr:
            tl, k, N = _glwe(self.params)
            sample = self.sample.to(thr.device)
            self._spectra = (thr, (thr.ntt_forward_i32(sample[:k].contiguous()), sample[k].contiguous()))
        return self._spectra[1]

    def dump(self, file_obj):
        pickle.dump(_KEY_TAG, file_obj)
        pickle.dump(self.params, file_obj)
        pickle.dump(self.n, file_obj)
        pickle.dump(self.sample.cpu().numpy(), file_obj)

    def dumps(self):
        file_obj = io.BytesIO()
        self.dump(file_obj)
        return file_obj.getvalue()

    @classmethod
    def load(cls, file_obj, thr):
        _check_tag(file_obj, _KEY_TAG)
        params, n, sample = _fields(file_obj, 3)
        if not isinstance(sample, numpy.ndarray) or sample.dtype != numpy.int32:
            raise ValueError('a damaged re-encryption key pickle')
        return cls(params, n, thr.to_device(sample))

    @classmethod
    def loads(cls, s: bytes, thr):
        return cls.load(io.BytesIO(s), thr)

    def __eq__(self, other):
        return (self.__class__ == other.__class__ and self.params == other.params and self.n == other.n
                and torch.equal(self.sample.cpu(), other.sample.cpu()))


def key_messages(secret_key, N):
    """The Torus32 messages (N,) of the key's slots: s_A[i] g_j at slot 2 i + j, 0 from slot 2 n on."""
    s = secret_key.lwe_key.key.reshape(-1).to(torch.int64)
    n = s.numel()
    mus = torch.zeros(N, dtype=torch.int64, device=s.device)
    for j, g in enumerate(GADGET):
        mus[j:LEVELS * n:LEVELS] = s * g
    return mus


def _wrap_i32(x):
    """int64 values -> their residues mod 2^32 as int32."""
    x = x & 0xffffffff
    return torch.where(x >= 1 << 31, x - (1 << 32), x).to(torch.int32)


def make_reencryption_key(thr, rng, secret_key, compact_public_key):
    """The re-encryption key from `secret_key` (the sender's NuFHESecretKey, s_A) to the owner of `compact_public_key`
    (the recipient's NuFHECompactPublicKey, a GLWE encryption of zero under S_B).  Draws the seed of r, then e1 (1, k, N)
    and e2 (1, N), as compact_encrypt does for one group; the sums are kept at 32 bits.

    Security:
      * The key is a compact public-key encryption under S_B, so it rests on the same assumption as the compact public
        key (DESIGN.md section 16) and creates no key cycle: it encrypts s_A, never S_B.
      * What the server does with it depends only on the number of rows it re-encrypts.
      * It is unidirectional: it moves ciphertexts from A to B, not back.
      * Anyone who holds both the key and S_B can decrypt it and recover s_A.  The server must never hand the key to B:
        a server that colludes with B learns all of A's data.  This is the trust model of key-switching proxy
        re-encryption; no attempt at collusion resistance is made.
      * A key made for the wrong recipient gives noise after re-encryption, not an error: nothing can check the
        recipient without secrets.

    TypeError unless given a NuFHESecretKey and a NuFHECompactPublicKey; ValueError when they were made for different
    parameters, or for parameters re-encryption does not take (k != 1, 2 n > N)."""
    from .api_low_level import NuFHESecretKey
    if not isinstance(secret_key, NuFHESecretKey):
        raise TypeError('make_reencryption_key needs the sender\'s NuFHESecretKey, got %s' % type(secret_key).__name__)
    if not isinstance(compact_public_key, NuFHECompactPublicKey):
        raise TypeError('make_reencryption_key needs the recipient\'s NuFHECompactPublicKey, got %s'
                        % type(compact_public_key).__name__)
    params = compact_public_key.params
    if secret_key.params != params:
        raise ValueError('the secret key and the compact public key were made for different parameters')
    tl, k, N = _glwe(params)
    n = params.in_out_params.size
    _check_shape(params, n)
    r_seed = draw_seed(rng)
    e1 = rand_gaussian_torus32(thr, rng, 0, tl.min_noise, (1, k, N))
    e2 = rand_gaussian_torus32(thr, rng, 0, tl.min_noise, (1, N))
    spec = thr.ntt_forward_i32(r_bits(thr, r_seed, 1, N)).reshape(1, 1, N)
    prod = thr.ntt_inverse_i32(thr.ntt_mac(spec, compact_public_key.spectra(thr)))[0].to(torch.int64)
    sample = prod.clone()
    sample[:k] += e1[0].to(prod.device, torch.int64)
    sample[k] += e2[0].to(prod.device, torch.int64) + key_messages(secret_key, N).to(prod.device)
    return NuFHEReencryptionKey(params, n, _wrap_i32(sample))


# ---------------------------------------------------------------- noise

def reencrypt_variance(params):
    """What re-encryption adds to a sample's phase before the key switch: the key term n t E[d^2] fresh (every slot's
    fresh compact noise times a digit, 2.89e-7 for the default parameters) and the 16-bit rounding of the input masks,
    each multiplied by a key bit, (n / 2) 2^-32 / 12 (4.9e-9)."""
    n = params.in_out_params.size
    fresh = noise_terms(params)[0]
    return n * LEVELS * DIGIT_SQUARE * fresh + n / 2 * 2.0**-32 / 12


def keyswitch_variance(params):
    """The cloud key's key switch (3.64e-6)."""
    return noise_terms(params)[3]


def output_lut_sigma(params, log2_outputs, shift=None):
    """Standard deviation of the rounded phase of a vm.lut input made of re-encrypted LUT outputs (index_lookup's rule,
    with the re-encryption and the second key switch as what the input carries beyond a LUT output)."""
    return index_lookup.lut_input_sigma(params, lut.bootstrap_variance(params) + reencrypt_variance(params), 0,
                                        log2_outputs, shift)


def margins(params):
    """{(bits, log2_outputs, shift): noise margin in sigma} of a re-encrypted LUT output for every lut.ALLOWED
    configuration."""
    return {(P, L, sh): 2.0**-(P + 2) / output_lut_sigma(params, L, sh) for P, L, sh in sorted(lut.ALLOWED, key=str)}


def max_input_variance(params):
    """The largest recorded variance of an input whose re-encryption still keeps lut.MARGIN_SIGMAS as one input of a
    two-input gate (box 1/8): the other input a gate output, and the blind-rotation term that current_variances does not
    record counted as lut does (lut.lut_sigma of two LUT outputs, shift 0)."""
    # a re-encrypted input of recorded variance v carries v + reencrypt_variance + the key switch, plus the unrecorded
    # blind-rotation term; beyond a gate output (blind rotation + key switch) that is v + reencrypt_variance
    return (0.125 / lut.MARGIN_SIGMAS)**2 - lut.lut_sigma(params, 0, 0)**2 - reencrypt_variance(params)


def _default_max_input_variance():
    from .api_low_level import NuFHEParameters
    return max_input_variance(NuFHEParameters())


MAX_INPUT_VARIANCE = _default_max_input_variance()


# ---------------------------------------------------------------- the server's work

def rows_per_pass(params):
    """Rows re-encrypted per pass: as many as keep the extracted masks (k N words per row) within compact.PASS_BYTES."""
    tl, k, N = _glwe(params)
    return max(1, PASS_BYTES // (k * N * 4))


def check_inputs(params, rekey, ciphertexts, tenant=None):
    where = '' if tenant is None else 'tenant %d: ' % tenant
    if not isinstance(rekey, NuFHEReencryptionKey):
        raise TypeError('%sreencrypt needs a NuFHEReencryptionKey (ctx.make_reencryption_key), got %s'
                        % (where, type(rekey).__name__))
    if rekey.params != params:
        raise ValueError('%sthe re-encryption key was made for other parameters than this machine' % where)
    if not isinstance(ciphertexts, LweSampleArray):
        raise TypeError('%sreencrypt needs an LweSampleArray, got %s' % (where, type(ciphertexts).__name__))
    if ciphertexts.a.shape[-1] != rekey.n:
        raise ValueError('%sthe ciphertexts have LWE dimension %d, the re-encryption key %d'
                         % (where, ciphertexts.a.shape[-1], rekey.n))
    if ciphertexts.current_variances.numel():
        worst = float(ciphertexts.current_variances.max())
        limit = max_input_variance(params)
        if worst > limit:
            raise ValueError('%sa ciphertext with variance %.3g is above the %.3g that re-encryption takes: bootstrap '
                             'it first' % (where, worst, limit))


def reencrypt_rows(thr, params, keys, rekeys, parts, out):
    """Re-encrypt the concatenation of `parts` ((a, b, variances) per segment, in order) with rekeys[i] for the rows of
    parts[i], then key-switch them with `keys` (batch_keys) into out = (a, b, variances), a few rows per pass: one
    nb_reencrypt launch with one segment per key, then one key switch, per pass."""
    counts = [p[1].numel() for p in parts]
    B = sum(counts)
    if B == 0:
        return
    n = rekeys[0].n
    a = torch.cat([p[0].reshape(-1, n) for p in parts]) if len(parts) > 1 else parts[0][0].reshape(-1, n)
    b = torch.cat([p[1].reshape(-1) for p in parts]) if len(parts) > 1 else parts[0][1].reshape(-1)
    cv = torch.cat([p[2].reshape(-1) for p in parts]) if len(parts) > 1 else parts[0][2].reshape(-1)
    spectra = [r.spectra(thr) for r in rekeys]
    out_a, out_b, out_cv = out[0].view(-1, out[0].shape[-1]), out[1].view(-1), out[2].view(-1)
    extra = reencrypt_variance(params)
    step = rows_per_pass(params)
    for r0 in range(0, B, step):
        r1 = min(B, r0 + step)
        idx, own = owners(counts, r0, r1)
        ext = thr.reencrypt(a[r0:r1], b[r0:r1], [spectra[i][0] for i in idx], [spectra[i][1] for i in idx], own)
        _, _, rcv = keys.split(r0, r1).keyswitch(ext, out=(out_a[r0:r1], out_b[r0:r1]), want_cv=True)
        del ext
        out_cv[r0:r1] = cv[r0:r1] + rcv + extra


def reencrypt(thr, params, ks, rekey, ciphertexts, dest=None):
    """VirtualMachine.reencrypt: the LweSampleArray, under the cloud key whose key switch is `ks`, of `ciphertexts`."""
    check_inputs(params, rekey, ciphertexts)
    if dest is not None and tuple(dest.shape) != tuple(ciphertexts.shape):
        raise ValueError('dest has shape %s, the ciphertexts %s' % (tuple(dest.shape), tuple(ciphertexts.shape)))
    out = dest if dest is not None else LweSampleArray.empty(thr, params.in_out_params, ciphertexts.shape)
    parts = [(ciphertexts.a, ciphertexts.b, ciphertexts.current_variances)]
    reencrypt_rows(thr, params, OneKey(thr, ks=ks), [rekey], parts, (out.a, out.b, out.current_variances))
    return out
