"""Compact public-key encryption (DESIGN.md section 16): a 5 KB ring public key, and ciphertexts of 4 bytes per bit that
the server expands into ordinary LWE samples.

The compact public key is one GLWE encryption of zero under the bootstrap key's GLWE key S (k polynomials of N = 1024
coefficients): masks A (k, N), the ChaCha20 stream (seed, nonce 7), and body B = A.S + E.  It stores the seed and B.

Encrypting B messages: message c (C order) goes to group g = c // N, slot p = c % N.  Per group, with r a fresh binary
polynomial (stream (r_seed, nonce 8) as (G, N / 32) words, bit i of group g = bit i % 32 of word (g, i // 32); r_seed
is drawn per call and never stored) and Gaussian noises e1 (G, k, N), e2 (G, N) of the bootstrap key's sigma,

    mask_u = A_u r + e1_u,    body = B r + e2 + sum_{c in g} mu_c X^p,

every coefficient rounded to 16 bits (packing's rounding), empty body slots stored as 0.  The products go through the
exact NTT: every coefficient of A_u r is below N 2^31 < p / 2 in magnitude.

Expansion (server): coefficient p of the restored sample (x << 16) is extracted into an LWE sample under the extracted
key of S, a'[u N + j] = A'_u[p - j] (j <= p) or -A'_u[N + p - j] (j > p), b' = body'[p], and the cloud key's key switch
takes it to the LWE key s.  The masks are multiples of 2^16, so the key switch's 16-bit digit cut rounds nothing."""
import io
import pickle

import numpy
import torch

from .lwe import LweSampleArray
from .tlwe import TLweSampleArray, tlwe_encrypt_zero_with_masks
from .compressed import draw_seed, _check_tag
from .random_numbers import rand_gaussian_torus32
from .batch_keys import OneKey, group_rows

NONCE_COMPACT_KEY = 7
NONCE_COMPACT_RANDOMNESS = 8
PASS_BYTES = 64 << 20                   # extracted masks of one expansion pass (a few groups), whatever the batch

_KEY_TAG = 'nufhe_b200.NuFHECompactPublicKey/1'
_CIPHERTEXT_TAG = 'nufhe_b200.CompactLweSampleArray/1'


def _glwe(params):
    tl = params.tgsw_params.tlwe_params
    return tl, tl.mask_size, tl.polynomial_degree


def groups_per_pass(params):
    """Groups expanded per pass: as many as keep the extracted masks (N rows of k N words per group) within
    PASS_BYTES (16 for k = 1)."""
    tl, k, N = _glwe(params)
    return max(1, PASS_BYTES // (N * k * N * 4))


def noise_terms(params):
    """Variances (torus units) of an expanded sample's phase: (fresh, mask rounding, body rounding, key switch).
    fresh: E.r + e2 - e1.S with r and S binary, about ((k + 1) N / 2 + 1) sigma^2; the 16-bit rounding of the k N mask
    coefficients, each multiplied by a key bit, (k N / 2) 2^-32 / 12, and of the body, 2^-32 / 12; the key switch,
    k N t (base - 1) / base ks_stdev^2 (DESIGN.md section 9)."""
    tl, k, N = _glwe(params)
    fresh = ((k + 1) * N / 2 + 1) * tl.min_noise**2
    rnd = 2.0**-32 / 12
    base = 2**params.ks_log2_base
    ks = k * N * params.ks_decomp_length * (base - 1) / base * params.in_out_params.min_noise**2
    return fresh, k * N / 2 * rnd, rnd, ks


class NuFHECompactPublicKey:
    """params, the 256-bit seed of the masks A (k, N) and the body B (N,) int32: 5.2 KB pickled for k = 1, 4 KB of it the body.
    `ctx.encrypt(cpk, bits)` and `ctx.encrypt_int(cpk, values, bits)` take it in place of the secret key and return a
    CompactLweSampleArray.  `spectra(thr)` -- the NTT of the k + 1 key polynomials -- is built once per engine and
    cached on the object."""

    def __init__(self, params, seed, b):
        self.params = params
        self.seed = numpy.asarray(seed, numpy.uint32).reshape(8)
        self.b = b
        tl, k, N = _glwe(params)
        if tuple(b.shape) != (N,):
            raise ValueError('a compact public key for these parameters has body shape %s, got %s' % ((N,), tuple(b.shape)))
        self._spectra = None

    @classmethod
    def from_tgsw_key(cls, thr, rng, params, tgsw_key):
        """A GLWE encryption of zero under the bootstrap key's GLWE key with seeded masks: draws the seed, then the
        Gaussian body noise E (N,)."""
        tl, k, N = _glwe(params)
        seed = draw_seed(rng)
        noise = rand_gaussian_torus32(thr, rng, 0, tl.min_noise, (N,))
        sample = TLweSampleArray.empty(thr, tl, ())
        tlwe_encrypt_zero_with_masks(thr, sample, _masks(thr, seed, params), noise, tl.min_noise, tgsw_key.tlwe_key)
        return cls(params, seed, sample.a.coeffs[k].contiguous())

    def masks(self, thr):
        """The masks A (k, N), regenerated from the seed."""
        return _masks(thr, self.seed, self.params)

    def spectra(self, thr):
        """NTT of the key polynomials (A_0, ..., A_{k-1}, B) as (1, k + 1, N) field elements: what nb_ntt_mac reads."""
        if self._spectra is None or self._spectra[0] is not thr:
            tl, k, N = _glwe(self.params)
            polys = torch.cat([self.masks(thr), self.b.to(thr.device)[None, :]], dim=0)
            self._spectra = (thr, thr.ntt_forward_i32(polys.contiguous()).reshape(1, k + 1, N))
        return self._spectra[1]

    def dump(self, file_obj):
        pickle.dump(_KEY_TAG, file_obj)
        pickle.dump(self.params, file_obj)
        pickle.dump(self.seed, file_obj)
        pickle.dump(self.b.cpu().numpy(), file_obj)

    def dumps(self):
        file_obj = io.BytesIO()
        self.dump(file_obj)
        return file_obj.getvalue()

    @classmethod
    def load(cls, file_obj, thr):
        _check_tag(file_obj, _KEY_TAG)
        params, seed, b = _fields(file_obj, 3)
        return cls(params, seed, thr.to_device(b))

    @classmethod
    def loads(cls, s: bytes, thr):
        return cls.load(io.BytesIO(s), thr)

    def __eq__(self, other):
        return (self.__class__ == other.__class__ and self.params == other.params and (self.seed == other.seed).all()
                and torch.equal(self.b.cpu(), other.b.cpu()))


def _fields(file_obj, count):
    """The next `count` pickled fields; ValueError for a truncated or damaged pickle."""
    try:
        return [pickle.load(file_obj) for _ in range(count)]
    except (pickle.UnpicklingError, EOFError) as e:
        raise ValueError('a truncated or damaged pickle: %s' % e) from e


def _masks(thr, seed, params):
    tl, k, N = _glwe(params)
    return thr.seeded_uniform(seed, NONCE_COMPACT_KEY, (k, N))


class CompactLweSampleArray:
    """Compact ciphertexts: params, the shape of the message array and `data` (G, k + 1, N) uint16, G = ceil(size / N).
    Pickled as the tag, params, shape and the data as little-endian uint16 bytes: 4 bytes per bit for k = 1.
    `vm.expand` turns it into an LweSampleArray of the same shape."""

    def __init__(self, params, shape, data):
        self.params = params
        self.shape = tuple(int(s) for s in shape)
        self.data = data
        tl, k, N = _glwe(params)
        want = (-(-self.size // N), k + 1, N)
        if tuple(data.shape) != want or data.dtype != torch.uint16:
            raise ValueError('compact data of %s items is uint16 %s, got %s %s'
                             % (self.shape, want, data.dtype, tuple(data.shape)))

    @property
    def size(self):
        return int(numpy.prod(self.shape, dtype=numpy.int64))

    def dump(self, file_obj):
        pickle.dump(_CIPHERTEXT_TAG, file_obj)
        pickle.dump(self.params, file_obj)
        pickle.dump(self.shape, file_obj)
        pickle.dump(self.data.cpu().numpy().astype('<u2').tobytes(), file_obj)

    def dumps(self):
        file_obj = io.BytesIO()
        self.dump(file_obj)
        return file_obj.getvalue()

    @classmethod
    def load(cls, file_obj, thr):
        _check_tag(file_obj, _CIPHERTEXT_TAG)
        params, shape, raw = _fields(file_obj, 3)
        shape = tuple(shape)
        tl, k, N = _glwe(params)
        groups = -(-int(numpy.prod(shape, dtype=numpy.int64)) // N)
        if not isinstance(raw, bytes) or len(raw) != groups * (k + 1) * N * 2:
            raise ValueError('compact data does not match shape %s' % (shape,))
        data = numpy.frombuffer(raw, '<u2').astype(numpy.uint16).reshape(groups, k + 1, N)
        return cls(params, shape, thr.to_device(data))

    @classmethod
    def loads(cls, s: bytes, thr):
        return cls.load(io.BytesIO(s), thr)

    def __eq__(self, other):
        return (self.__class__ == other.__class__ and self.params == other.params and self.shape == other.shape
                and numpy.array_equal(self.data.cpu().numpy(), other.data.cpu().numpy()))


def r_bits(thr, r_seed, groups, N=1024):
    """The binary polynomials r (G, N) int32 of one encryption: bit i of group g = bit i % 32 of word (g, i // 32) of
    the stream (r_seed, nonce 8)."""
    words = thr.seeded_uniform(r_seed, NONCE_COMPACT_RANDOMNESS, (groups, N // 32))
    shifts = torch.arange(32, dtype=torch.int32, device=words.device)
    return ((words[:, :, None] >> shifts) & 1).reshape(groups, N).contiguous()


def compact_encrypt(thr, rng, cpk: NuFHECompactPublicKey, mus):
    """Encrypt the Torus32 messages `mus` (a device int32 tensor of any shape) with the compact public key.  Draws the
    seed of r, then e1 (G, k, N) and e2 (G, N)
    (nb_ntt_forward_i32 -> nb_ntt_mac -> nb_ntt_inverse_i32 -> nb_compact_finish)."""
    params = cpk.params
    tl, k, N = _glwe(params)
    shape = tuple(mus.shape)
    batch = int(numpy.prod(shape, dtype=numpy.int64))
    groups = -(-batch // N)
    r_seed = draw_seed(rng)
    e1 = rand_gaussian_torus32(thr, rng, 0, tl.min_noise, (groups, k, N))
    e2 = rand_gaussian_torus32(thr, rng, 0, tl.min_noise, (groups, N))
    if groups == 0:
        return CompactLweSampleArray(params, shape, thr.empty((0, k + 1, N), torch.uint16))
    spec = thr.ntt_forward_i32(r_bits(thr, r_seed, groups, N)).reshape(groups, 1, N)
    prod = thr.ntt_inverse_i32(thr.ntt_mac(spec, cpk.spectra(thr)))
    return CompactLweSampleArray(params, shape, thr.compact_finish(prod, e1, e2, mus.reshape(-1)))


def expand(thr, params, ks, compact: CompactLweSampleArray):
    """The LweSampleArray (under the cloud key's LWE key s) of a CompactLweSampleArray, a few groups per pass
    (nb_compact_extract -> nb_keyswitch with `ks`, the cloud key's LweKeyswitchKey).  Its variances are the key
    switch's plus the fresh and rounding terms of noise_terms."""
    out = LweSampleArray.empty(thr, params.in_out_params, compact.shape)
    expand_groups(thr, params, OneKey(thr, ks=ks), [compact], (out.a, out.b, out.current_variances))
    return out


def expand_groups(thr, params, keys, compacts, out):
    """Expand `compacts`, one CompactLweSampleArray per tenant of `keys` (batch_keys), into the concatenation of their
    rows, out = (a, b, variances), a few groups per pass.  One tenant's rows are extracted and key-switched straight
    into `out`; with several, whole groups are extracted and the slots that pad a tenant's last group are dropped."""
    tl, k, N = _glwe(params)
    a, b, cv = out[0].view(-1, out[0].shape[-1]), out[1].view(-1), out[2].view(-1)
    fresh, mask_rnd, body_rnd, _ = noise_terms(params)
    if len(compacts) == 1:
        data, B = compacts[0].data.to(thr.device), compacts[0].size
        G = -(-B // N)
    else:
        groups, rows = group_rows(keys.counts, N, -1)
        data, G = torch.cat([c.data.to(thr.device) for c in compacts]), sum(groups)
    step = groups_per_pass(params)
    for p0 in range(0, G, step):
        p1 = min(G, p0 + step)
        if len(compacts) == 1:
            r0, r1 = p0 * N, min(B, p1 * N)
            ext = thr.compact_extract(data[p0:p1], r1 - r0)
        else:
            slots = rows[p0 * N:p1 * N]
            real = numpy.nonzero(slots >= 0)[0]
            r0, r1 = int(slots[real[0]]), int(slots[real[-1]]) + 1      # the rows of a pass are consecutive
            ext = thr.compact_extract(data[p0:p1], (p1 - p0) * N)
            if len(real) < len(slots):
                sel = thr.to_device(real)
                ext = ext[0].index_select(0, sel), ext[1].index_select(0, sel)
        _, _, rcv = keys.split(r0, r1).keyswitch(ext, out=(a[r0:r1], b[r0:r1]), want_cv=True)
        del ext
        cv[r0:r1] = rcv + (fresh + mask_rnd + body_rnd)
