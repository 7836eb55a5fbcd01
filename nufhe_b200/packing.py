"""Result packing (DESIGN.md section 12): up to N = 1024 LWE samples under the LWE key s (n words) become one GLWE sample
under a fresh binary GLWE key S_p (k polynomials of N coefficients), rounded to 16 bits per coefficient, so that
results download at 4 bytes per bit instead of about 2 KB.

The packing key K holds n t GLWE encryptions under S_p: K_ij encrypts the constant polynomial s_i g_j, with the fixed
decomposition t = 2 levels of base 2^8, g_0 = 2^24, g_1 = 2^16.  It is stored seeded: its masks are the ChaCha20 stream
(seed, nonce 4) of shape (n, t, k, N), and it keeps the bodies body_ij = e_ij + sum_u A_iju S_p,u + s_i g_j X^0.

Packing B inputs: input c (C order) goes to group g = c // N, slot p = c % N; with the digits d_cij of a_ci
(pack_layout.cuh), D_gij = sum_{c in g} d_cij X^p and C_gu = sum_ij D_gij K_iju (negacyclic, mod 2^32, computed through
the exact NTT), the packed sample is (-C_g0, ..., -C_g,k-1, sum_{c in g} b_c X^p - C_gk), every coefficient rounded to
its top 16 bits.  Coefficient p of its phase under S_p is the phase of input c."""
import io
import pickle

import numpy
import torch

from .lwe import LweSampleArray
from .tlwe import TLweKey, TLweSampleArray, tlwe_encrypt_zero_with_masks
from .polynomials import IntPolynomialArray
from .compressed import draw_seed, _check_tag, _variance, _wrap32
from .random_numbers import rand_gaussian_torus32
from .batch_keys import OneKey, group_rows

NONCE_PACKING_KEY = 4
PACK_LEVELS = 2                         # t
PACK_LOG2_BASE = 8
PACK_GADGET = (2**24, 2**16)            # g_j = 2^(32 - (j + 1) * 8)
PACK_BITS = 16                          # bits kept per output coefficient
PASS_SPECTRA_BYTES = 64 << 20           # digit spectra of one packing pass (a few groups), whatever the batch

_SECRET_KEY_TAG = 'nufhe_b200.NuFHEPackingSecretKey/1'
_PACKING_KEY_TAG = 'nufhe_b200.NuFHEPackingKey/1'
_PACKED_TAG = 'nufhe_b200.PackedLweSampleArray/1'


def _glwe(params):
    tl = params.tgsw_params.tlwe_params
    return tl, tl.mask_size, tl.polynomial_degree


def groups_per_pass(params):
    """Groups packed per pass: as many as keep the (groups, n t, N) digit spectra within PASS_SPECTRA_BYTES (8 for the
    default parameters)."""
    tl, k, N = _glwe(params)
    per_group = params.in_out_params.size * PACK_LEVELS * N * 8
    return max(1, PASS_SPECTRA_BYTES // per_group)


class NuFHEPackingSecretKey:
    """The client's half of a packing key pair: params and the binary GLWE key S_p (k, N) int32.  Decrypts
    PackedLweSampleArray results (`ctx.decrypt`, `ctx.decrypt_int`); kept next to the NuFHESecretKey."""

    def __init__(self, params, key):
        self.params = params
        self.key = key
        tl, k, N = _glwe(params)
        if tuple(key.shape) != (k, N):
            raise ValueError('a packing secret key for these parameters has shape %s, got %s' % ((k, N), tuple(key.shape)))

    @classmethod
    def from_rng(cls, thr, params, rng):
        """S_p drawn like a TGSW key (TLweKey.from_rng: k N uniform bits)."""
        return cls(params, TLweKey.from_rng(thr, params.tgsw_params.tlwe_params, rng).key.coeffs)

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


class _GadgetKey:
    """n t seeded GLWE encryptions of the constants s_i g_j (s the LWE key, g_j = PACK_GADGET[j]) under a GLWE key:
    params, the 256-bit seed of the masks (ChaCha20 stream (seed, NONCE)), the bodies (n, t, N) int32 and the variance
    of their noise.  The packing key and the tree key (nufhe_b200/tree_lut.py) are two distinct subclasses.
    `spectra(thr)` -- the NTT of all n t (k+1) key polynomials, 16.4 MB for k = 1 -- is built once per engine and cached
    on the object: with it, `pack` packs under the key's GLWE key (S_p for the packing key, S for the tree key)."""
    NONCE = None
    TAG = None
    NAME = None

    def __init__(self, params, seed, body, variance: float):
        self.params = params
        self.seed = numpy.asarray(seed, numpy.uint32).reshape(8)
        self.body = body
        self.variance = float(variance)
        self._spectra = None
        tl, k, N = _glwe(params)
        want = (params.in_out_params.size, PACK_LEVELS, N)
        if tuple(body.shape) != want:
            raise ValueError('a %s for these parameters has body shape %s, got %s' % (self.NAME, want, tuple(body.shape)))

    @classmethod
    def _encrypt(cls, thr, rng, secret_key, glwe_key):
        """K_ij = GLWE_{glwe_key}(s_i g_j) with seeded masks: draws the seed, then the Gaussian body noises (n, t, N)."""
        params = secret_key.params
        tl, k, N = _glwe(params)
        n = params.in_out_params.size
        seed = draw_seed(rng)
        noises = rand_gaussian_torus32(thr, rng, 0, tl.min_noise, (n, PACK_LEVELS, N))
        samples = TLweSampleArray.empty(thr, tl, (n, PACK_LEVELS))
        key = TLweKey(tl, IntPolynomialArray(glwe_key))
        tlwe_encrypt_zero_with_masks(thr, samples, _masks(thr, seed, params, cls.NONCE), noises, tl.min_noise, key)
        body = samples.a.coeffs[..., k, :].contiguous()
        g = torch.tensor(PACK_GADGET, dtype=torch.int64, device=body.device)
        msg = secret_key.lwe_key.key.to(body.device).to(torch.int64)[:, None] * g[None, :]      # (n, t): s_i g_j
        body[:, :, 0] = _wrap32((body[:, :, 0].to(torch.int64) + msg) & 0xffffffff)
        return cls(params, seed, body, _variance(tl.min_noise))

    def masks(self, thr):
        """The masks A (n, t, k, N), regenerated from the seed."""
        return _masks(thr, self.seed, self.params, self.NONCE)

    def spectra(self, thr):
        """NTT of the key polynomials K_iju as (n t, k + 1, N) field elements, row i t + j: what nb_ntt_mac reads."""
        if self._spectra is None or self._spectra[0] is not thr:
            tl, k, N = _glwe(self.params)
            polys = torch.cat([self.masks(thr), self.body.to(thr.device)[:, :, None, :]], dim=2)   # (n, t, k+1, N)
            spec = thr.ntt_forward_i32(polys.contiguous()).reshape(-1, k + 1, N)
            self._spectra = (thr, spec)
        return self._spectra[1]

    def dump(self, file_obj):
        pickle.dump(self.TAG, file_obj)
        pickle.dump(self.params, file_obj)
        pickle.dump(self.seed, file_obj)
        pickle.dump(self.body.cpu().numpy(), file_obj)
        pickle.dump(self.variance, file_obj)

    def dumps(self):
        file_obj = io.BytesIO()
        self.dump(file_obj)
        return file_obj.getvalue()

    @classmethod
    def load(cls, file_obj, thr):
        _check_tag(file_obj, cls.TAG)
        params = pickle.load(file_obj)
        seed = pickle.load(file_obj)
        body = thr.to_device(pickle.load(file_obj))
        variance = pickle.load(file_obj)
        return cls(params, seed, body, variance)

    @classmethod
    def loads(cls, s: bytes, thr):
        return cls.load(io.BytesIO(s), thr)

    def __eq__(self, other):
        return (self.__class__ == other.__class__ and self.params == other.params and (self.seed == other.seed).all()
                and torch.equal(self.body.cpu(), other.body.cpu()) and self.variance == other.variance)


class NuFHEPackingKey(_GadgetKey):
    """The server's half: params, the 256-bit seed of the masks, the bodies (n, t, N) int32 (4.1 MB for the default
    parameters) and the variance of their noise."""
    NONCE = NONCE_PACKING_KEY
    TAG = _PACKING_KEY_TAG
    NAME = 'packing key'

    @classmethod
    def from_secret_key(cls, thr, rng, secret_key, packing_secret_key: NuFHEPackingSecretKey):
        """K_ij = GLWE_{S_p}(s_i g_j) with seeded masks: draws the seed, then the Gaussian body noises (n, t, N)."""
        return cls._encrypt(thr, rng, secret_key, packing_secret_key.key)


def _masks(thr, seed, params, nonce=NONCE_PACKING_KEY):
    tl, k, N = _glwe(params)
    return thr.seeded_uniform(seed, nonce, (params.in_out_params.size, PACK_LEVELS, k, N))


class PackedLweSampleArray:
    """Packed results: params, the shape of the packed array and `data` (G, k + 1, N) uint16, G = ceil(size / N).
    Pickled as the tag, params, shape and the data as little-endian uint16 bytes: 4 bytes per bit for k = 1."""

    def __init__(self, params, shape, data):
        self.params = params
        self.shape = tuple(int(s) for s in shape)
        self.data = data
        tl, k, N = _glwe(params)
        want = (-(-self.size // N), k + 1, N)
        if tuple(data.shape) != want or data.dtype != torch.uint16:
            raise ValueError('packed data of %s items is uint16 %s, got %s %s'
                             % (self.shape, want, data.dtype, tuple(data.shape)))

    @property
    def size(self):
        return int(numpy.prod(self.shape, dtype=numpy.int64))

    def dump(self, file_obj):
        pickle.dump(_PACKED_TAG, file_obj)
        pickle.dump(self.params, file_obj)
        pickle.dump(self.shape, file_obj)
        pickle.dump(self.data.cpu().numpy().astype('<u2').tobytes(), file_obj)

    def dumps(self):
        file_obj = io.BytesIO()
        self.dump(file_obj)
        return file_obj.getvalue()

    @classmethod
    def load(cls, file_obj, thr):
        _check_tag(file_obj, _PACKED_TAG)
        params = pickle.load(file_obj)
        shape = tuple(pickle.load(file_obj))
        raw = pickle.load(file_obj)
        tl, k, N = _glwe(params)
        groups = -(-int(numpy.prod(shape, dtype=numpy.int64)) // N)
        if not isinstance(raw, bytes) or len(raw) != groups * (k + 1) * N * 2:
            raise ValueError('packed data does not match shape %s' % (shape,))
        data = numpy.frombuffer(raw, '<u2').astype(numpy.uint16).reshape(groups, k + 1, N)
        return cls(params, shape, thr.to_device(data))

    @classmethod
    def loads(cls, s: bytes, thr):
        return cls.load(io.BytesIO(s), thr)

    def __eq__(self, other):
        return (self.__class__ == other.__class__ and self.params == other.params and self.shape == other.shape
                and numpy.array_equal(self.data.cpu().numpy(), other.data.cpu().numpy()))


def make_packing_keys(thr, rng, secret_key):
    """(NuFHEPackingSecretKey, NuFHEPackingKey) for `secret_key`.  Draws S_p, then the seed, then the body noises."""
    psk = NuFHEPackingSecretKey.from_rng(thr, secret_key.params, rng)
    return psk, NuFHEPackingKey.from_secret_key(thr, rng, secret_key, psk)


def pack(thr, packing_key: _GadgetKey, ciphertexts: LweSampleArray):
    """Pack an LweSampleArray of any shape into a PackedLweSampleArray under the key's GLWE key, a few groups per pass
    (nb_pack_digits -> nb_ntt_forward_i32 -> nb_ntt_mac -> nb_ntt_inverse_i32 -> nb_pack_finish)."""
    params = packing_key.params
    if ciphertexts.params != params.in_out_params:
        raise ValueError('the ciphertexts do not have the LWE parameters of the packing key')
    tl, k, N = _glwe(params)
    n = params.in_out_params.size
    shape = tuple(ciphertexts.shape)
    batch = int(numpy.prod(shape, dtype=numpy.int64))
    if batch == 0:
        return PackedLweSampleArray(params, shape, thr.empty((0, k + 1, N), torch.uint16))
    keys = OneKey(thr, spectra=packing_key.spectra(thr))
    return PackedLweSampleArray(params, shape, pack_groups(thr, params, keys, [(ciphertexts.a.reshape(batch, n),
                                                                                 ciphertexts.b.reshape(batch))]))


def pack_groups(thr, params, keys, parts):
    """The packed groups (G, k + 1, N) uint16 of `parts`, one (a (c, n), b (c,)) per tenant of `keys` (batch_keys),
    each starting at a group boundary, so a group never mixes tenants.  One part is packed in slices of itself; several
    are gathered with a zero row in the slots that pad a tenant's last group, which packs exactly as an empty slot."""
    tl, k, N = _glwe(params)
    if len(parts) == 1:
        (a, b), = parts
        G = -(-b.shape[0] // N)
    else:
        counts = [b.shape[0] for a, b in parts]
        groups, src = group_rows(counts, N, sum(counts))          # padding: the zero row after the last part
        G, n = sum(groups), parts[0][0].shape[1]
        a_all = torch.cat([a for a, b in parts] + [thr.empty((1, n), torch.int32).zero_()])
        b_all = torch.cat([b for a, b in parts] + [thr.empty((1,), torch.int32).zero_()])
        src = thr.to_device(src)
    step = groups_per_pass(params)
    out = None if len(parts) == 1 and 0 < G <= step else thr.empty((G, k + 1, N), torch.uint16)
    for g0 in range(0, G, step):
        g1 = min(G, g0 + step)
        if len(parts) == 1:
            xa, xb = a[g0 * N:g1 * N].contiguous(), b[g0 * N:g1 * N].contiguous()
        else:
            idx = src[g0 * N:g1 * N]
            xa, xb = a_all.index_select(0, idx), b_all.index_select(0, idx)
        spec = thr.ntt_forward_i32(thr.pack_digits(xa))
        part = thr.pack_finish(thr.ntt_inverse_i32(keys.split(g0, g1).ntt_mac(spec)), xb)
        del spec
        if out is None:
            out = part
        else:       # (uint16 tensors are copied through their int16 view)
            out.view(torch.int16)[g0:g1].copy_(part.view(torch.int16))
    return out


def _check_pair(secret_key, packed):
    if not isinstance(secret_key, NuFHEPackingSecretKey) or not isinstance(packed, PackedLweSampleArray):
        raise TypeError('packed results are decrypted with a NuFHEPackingSecretKey (got %s and %s)'
                        % (type(secret_key).__name__, type(packed).__name__))
    if secret_key.params != packed.params:
        raise ValueError('the packing secret key and the packed results have different parameters')


def packed_phases(thr, secret_key: NuFHEPackingSecretKey, packed: PackedLweSampleArray):
    """The phases (Torus32, host array of the packed shape): phase_g = out_gk - sum_{u<k} out_gu S_p,u with every
    coefficient shifted back by 16 bits; coefficient p of group g is the phase of input g N + p."""
    _check_pair(secret_key, packed)
    tl, k, N = _glwe(packed.params)
    x = (packed.data.to(thr.device).view(torch.int16).to(torch.int64) & 0xffff) << PACK_BITS
    x = _wrap32(x)                                                                      # (G, k+1, N)
    key = thr.ntt_forward_i32(secret_key.key.to(thr.device).contiguous()).reshape(k, 1, N)
    ms = thr.ntt_inverse_i32(thr.ntt_mac(thr.ntt_forward_i32(x[:, :k].contiguous()), key))[:, 0]
    phase = _wrap32((x[:, k].to(torch.int64) - ms.to(torch.int64)) & 0xffffffff)
    return phase.reshape(-1)[:packed.size].reshape(packed.shape).cpu().numpy()


def decrypt_packed(thr, secret_key, packed):
    """Bits of packed gate outputs (t32_to_bool of the phases), in the packed shape."""
    from .api_low_level import t32_to_bool
    return t32_to_bool(packed_phases(thr, secret_key, packed))


def decrypt_packed_int(thr, secret_key, packed, bits):
    """Integers in [0, 2^bits) of packed integer results (lut.decode_int of the phases)."""
    from .lut import decode_int
    return decode_int(packed_phases(thr, secret_key, packed), bits)
