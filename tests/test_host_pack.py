"""Result packing on the CPU: the digit, slot and rounding functions of csrc/pack_layout.cuh (through the host
emulator) against the NumPy restatement (pack_ref.py), and the Python layer (nufhe_b200/packing.py) on the oracle-backed
engine double: draw order, the phase of every packing-key row, pack-then-decrypt round trips bit-exact against the
restatement, pickles, argument errors, and the exactness and noise figures of DESIGN.md section 12."""
import ctypes
import io
import os

import numpy
import pytest

import nufhe_b200
from nufhe_b200 import packing
from nufhe_b200.packing import NONCE_PACKING_KEY, PACK_GADGET, PACK_LEVELS
from nufhe_b200.random_numbers import DeterministicRNG
from chacha_ref import seeded_uniform
from fake_engine import FakeEngine, _np, _t
from oracle import oracle as O
import pack_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 0xffffffff00000001
SIGMA = 9e-9 * (2 / numpy.pi)**0.5
BOUNDARY = numpy.array([0, 2**15 - 1, 2**15, 0x7fff8000, 0xffff8000, -1, 2**31], numpy.int64)


@pytest.fixture(scope='module')
def emul():
    path = os.path.join(ROOT, 'nufhe_b200', 'csrc', 'libnb_host_emul.so')
    if not os.path.exists(path):
        import __graft_entry__ as g
        g.build()
    lib = ctypes.CDLL(path)
    for name in ('emul_pack_digits', 'emul_pack_round16', 'emul_pack_unround16'):
        getattr(lib, name).argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
        getattr(lib, name).restype = None
    lib.emul_pack_slot.argtypes = [ctypes.c_uint64, ctypes.c_void_p, ctypes.c_void_p]
    lib.emul_pack_slot.restype = None
    return lib


def _words(extra=4096, seed=1):
    rnd = numpy.random.RandomState(seed).randint(-2**31, 2**31, size=extra, dtype=numpy.int64)
    return pack_ref.i32(numpy.concatenate([BOUNDARY, BOUNDARY + 1, BOUNDARY - 1, rnd]))


def test_header_digits_match_the_restatement(emul):
    a = _words()
    got = numpy.empty((a.size, 2), numpy.int32)
    emul.emul_pack_digits(a.ctypes.data, a.size, got.ctypes.data)
    want = pack_ref.digits(a)
    assert (got == want).all()
    assert got.min() >= -128 and got.max() <= 127
    # sum_j d_j g_j = round_16(a) mod 2^32
    recon = pack_ref.u32(got[:, 0].astype(numpy.int64) * PACK_GADGET[0] + got[:, 1].astype(numpy.int64) * PACK_GADGET[1])
    assert (recon == (pack_ref.u32(a.astype(numpy.int64) + 2**15) & 0xffff0000)).all()
    assert (got[:len(BOUNDARY)] == [[0, 0], [0, 0], [0, 1], [-128, 0], [0, 0], [0, 0], [-128, 0]]).all()


def test_header_rounding_matches_the_restatement(emul):
    x = _words().view(numpy.uint32).copy()
    got = numpy.empty(x.size, numpy.uint16)
    emul.emul_pack_round16(x.ctypes.data, x.size, got.ctypes.data)
    assert (got == pack_ref.round16(x)).all()
    assert list(got[:len(BOUNDARY)]) == [0, 0, 1, 0x8000, 0, 0, 0x8000]
    back = numpy.empty(x.size, numpy.uint32)
    emul.emul_pack_unround16(got.ctypes.data, got.size, back.ctypes.data)
    assert (back.view(numpy.int32) == pack_ref.unround16(got)).all()
    err = (x.astype(numpy.int64) - back.astype(numpy.int64) + 2**31) % 2**32 - 2**31
    assert err.min() >= -2**15 and err.max() < 2**15


def test_header_slot_mapping(emul):
    g, p = ctypes.c_uint64(), ctypes.c_uint32()
    for c in (0, 1, 1023, 1024, 1025, 4095, 5000, 2**40 + 7):
        emul.emul_pack_slot(c, ctypes.byref(g), ctypes.byref(p))
        assert (g.value, p.value) == (c // 1024, c % 1024)


def test_exactness_bound():
    """Every coefficient of C_gu is at most n t N 128 2^31 < 2^58 < p / 2 in magnitude, so the forward NTT, the field
    MAC and the centred inverse give it exactly mod 2^32; decryption's products are bounded by k N 2^31."""
    for k in (1, 2):
        params = nufhe_b200.NuFHEParameters(tlwe_mask_size=k)
        n, N = params.in_out_params.size, params.tgsw_params.tlwe_params.polynomial_degree
        bound = n * PACK_LEVELS * N * 128 * 2**31
        assert bound < 2**58 < P // 2
        assert k * N * 2**31 < P // 2
    assert PACK_GADGET == (2**24, 2**16) and packing.PACK_LOG2_BASE == 8


def test_noise_estimate_figures():
    """The DESIGN.md section 12 figures for k = 1 from the parameters (pack_ref.noise_terms)."""
    key, rnd, ms = pack_ref.noise_terms(nufhe_b200.NuFHEParameters())
    assert abs(key - 2.9e-7) < 0.05e-7 and abs(rnd - 4.9e-9) < 0.05e-9 and abs(ms - 1.0e-8) < 0.05e-8
    assert key + rnd + ms < 3.1e-7


# ---------------------------------------------------------------- the Python layer on the engine double

class PackingFakeEngine(FakeEngine):
    """FakeEngine with Engine.seeded_uniform from the NumPy keystream, and Engine.pack_digits / ntt_mac / pack_finish
    (nb_pack_digits, nb_ntt_mac, nb_pack_finish) restated with NumPy and the oracle's field operations."""

    def seeded_uniform(self, seed, nonce, shape, first=0):
        return _t(seeded_uniform(seed, nonce, shape, first))

    def pack_digits(self, a):
        self._count('pack_digits')
        an = _np(a).astype(numpy.int64)
        batch, n = an.shape
        groups = -(-batch // 1024)
        w = (an + 0x80808000) & 0xffffffff
        d = numpy.stack([(w >> 24) - 128, ((w >> 16) & 255) - 128], -1).reshape(batch, 2 * n)
        out = numpy.zeros((groups * 1024, 2 * n), numpy.int32)
        out[:batch] = d
        return _t(out.reshape(groups, 1024, 2 * n).transpose(0, 2, 1))

    def ntt_mac(self, x, key):
        self._count('ntt_mac')
        xn, kn = _np(x, True) % numpy.uint64(O.P), _np(key, True) % numpy.uint64(O.P)
        G, R, N = xn.shape
        U = kn.shape[1]
        acc = numpy.zeros((G, U, N), numpy.uint64)
        for r in range(R):
            prod = O.ff_mul(numpy.broadcast_to(xn[:, r:r + 1], (G, U, N)), numpy.broadcast_to(kn[r][None], (G, U, N)))
            acc = O.ff_add(acc, prod)
        return _t(acc)

    def pack_finish(self, c, b):
        self._count('pack_finish')
        v = -_np(c).astype(numpy.int64)
        bn = _np(b).astype(numpy.int64).reshape(-1)
        G, k1, N = v.shape
        body = numpy.zeros(G * N, numpy.int64)
        body[:bn.size] = bn
        v[:, k1 - 1, :] += body.reshape(G, N)
        return _t(((((v & 0xffffffff) + 0x8000) >> 16) & 0xffff).astype(numpy.uint16))


def _context(seed):
    return nufhe_b200.Context(rng=DeterministicRNG(seed), thread=PackingFakeEngine())


def _key_polys(pk):
    k = pk.params.tgsw_params.tlwe_params.mask_size
    return pack_ref.key_polys(seeded_uniform(pk.seed, NONCE_PACKING_KEY, (500, PACK_LEVELS, k, 1024)), _np(pk.body))


def _keys(seed, k):
    ctx = _context(seed)
    sk = ctx.make_secret_key(tlwe_mask_size=k)
    psk, pk = ctx.make_packing_keys(sk)
    return ctx, sk, psk, pk


@pytest.fixture(scope='module')
def keys():
    return _keys(61, 1)


@pytest.fixture(scope='module')
def keys2():
    return _keys(62, 2)


@pytest.mark.parametrize('k', [1, 2])
def test_key_generation_draw_order_and_row_phases(keys, keys2, k):
    ctx, sk, psk, pk = keys if k == 1 else keys2
    seed = 61 if k == 1 else 62
    replay = DeterministicRNG(seed)
    s = replay.uniform_bool((500,))
    S = replay.uniform_bool((k, 1024))
    pseed = replay.uniform_torus32((8,)).view(numpy.uint32)
    e = O.double_to_t32(replay.gauss((500, PACK_LEVELS, 1024), SIGMA)).astype(numpy.int64)
    assert (_np(sk.lwe_key.key) == s).all() and (_np(psk.key) == S).all() and (pk.seed == pseed).all()
    assert tuple(pk.body.shape) == (500, 2, 1024) and pk.variance == float(numpy.float32(SIGMA**2))
    K = _key_polys(pk)                                                  # (n t, k+1, N)
    phase = pack_ref.u32(K[:, k].astype(numpy.int64))
    for u in range(k):
        M = pack_ref.negacyclic_matrix(S[u])
        x = pack_ref.u32(K[:, u])
        phase = pack_ref.u32(phase - ((x & 0xffff).astype(numpy.float64) @ M).astype(numpy.int64)
                             - (((x >> 16).astype(numpy.float64) @ M).astype(numpy.int64) << 16))
    msg = numpy.zeros((500, PACK_LEVELS, 1024), numpy.int64)
    msg[:, :, 0] = s[:, None].astype(numpy.int64) * numpy.array(PACK_GADGET)[None, :]
    err = pack_ref.i32(phase.reshape(500, PACK_LEVELS, 1024) - msg).astype(numpy.int64)
    assert (err == e).all()                                             # s_i g_j + e_ij exactly
    assert numpy.abs(err).max() < 8 * SIGMA * 2**32
    # a second context with the same seed reproduces both keys
    _, _, psk2, pk2 = _keys(seed, k)
    assert psk2 == psk and pk2 == pk


def _lwe_phase(sk, ct):
    key = _np(sk.lwe_key.key).astype(numpy.int64)
    return pack_ref.i32(_np(ct.b).astype(numpy.int64) - (_np(ct.a).astype(numpy.int64) * key).sum(-1))


def _check_packed(ctx, sk, psk, pk, ct):
    packed = packing.pack(ctx.thread, pk, ct)
    a, b = _np(ct.a).reshape(-1, 500), _np(ct.b).reshape(-1)
    assert packed.shape == tuple(ct.shape)
    assert (_np(packed.data) == pack_ref.pack(a, b, _key_polys(pk))).all()
    ph = packing.packed_phases(ctx.thread, psk, packed)
    assert ph.shape == tuple(ct.shape)
    assert (ph.reshape(-1) == pack_ref.phases(_np(packed.data), _np(psk.key))[:b.size]).all()
    diff = pack_ref.i32(ph.astype(numpy.int64) - _lwe_phase(sk, ct).astype(numpy.int64)).astype(numpy.int64)
    assert numpy.abs(diff).max() < 2**32 * 7 * 3.0e-7**0.5
    return packed


@pytest.mark.parametrize('shape', [(1,), (1023,), (1024,), (1025,), (3, 700)])
def test_pack_and_decrypt_bits(keys, shape):
    ctx, sk, psk, pk = keys
    bits = numpy.random.RandomState(len(shape) + sum(shape)).randint(0, 2, size=shape).astype(bool)
    packed = _check_packed(ctx, sk, psk, pk, ctx.encrypt(sk, bits))
    assert tuple(packed.data.shape) == (-(-bits.size // 1024), 2, 1024)
    got = ctx.decrypt(psk, packed)
    assert got.shape == bits.shape and (got == bits).all()


@pytest.mark.parametrize('shape', [(1025,), (3, 700)])
def test_pack_and_decrypt_2bit_integers(keys, shape):
    ctx, sk, psk, pk = keys
    values = numpy.random.RandomState(5).randint(0, 4, size=shape)
    packed = _check_packed(ctx, sk, psk, pk, ctx.encrypt_int(sk, values, 2))
    assert (ctx.decrypt_int(psk, packed, 2) == values).all()


def test_pack_and_decrypt_k2(keys2):
    ctx, sk, psk, pk = keys2
    bits = numpy.random.RandomState(7).randint(0, 2, size=1100).astype(bool)
    packed = _check_packed(ctx, sk, psk, pk, ctx.encrypt(sk, bits))
    assert tuple(packed.data.shape) == (2, 3, 1024)
    assert (ctx.decrypt(psk, packed) == bits).all()


def test_pickles(keys):
    ctx, sk, psk, pk = keys
    bits = numpy.arange(1030) % 3 == 0
    packed = packing.pack(ctx.thread, pk, ctx.encrypt(sk, bits))
    s = packed.dumps()
    assert len(s) <= 2 * 2 * 1024 * 2 + 1024
    back = ctx.load_packed_ciphertext(s)
    assert back == packed and ctx.load_packed_ciphertext(io.BytesIO(s)) == packed
    assert (ctx.decrypt(psk, back) == bits).all()
    assert ctx.load_packing_key(pk.dumps()) == pk and ctx.load_packing_key(io.BytesIO(pk.dumps())) == pk
    assert ctx.load_packing_secret_key(psk.dumps()) == psk
    assert ctx.load_packing_secret_key(io.BytesIO(psk.dumps())) == psk
    assert ctx.load_secret_key(sk.dumps()) == sk                  # the NuFHESecretKey pickle is unchanged
    loaders = (ctx.load_packed_ciphertext, ctx.load_packing_key, ctx.load_packing_secret_key)
    pickles = (s, pk.dumps(), psk.dumps())
    for i, load in enumerate(loaders):
        for j, wrong in enumerate(pickles + (sk.dumps(), ctx.encrypt(sk, [True], compressed=True).dumps(), b'junk')):
            if i != j:
                with pytest.raises(ValueError):
                    load(wrong)


def test_mismatched_keys_and_params(keys, keys2):
    ctx, sk, psk, pk = keys
    ctx2, sk2, psk2, pk2 = keys2
    ct = ctx.encrypt(sk, [True, False])
    packed = packing.pack(ctx.thread, pk, ct)
    with pytest.raises(TypeError):
        ctx.decrypt(sk, packed)
    with pytest.raises(TypeError):
        ctx.decrypt(psk, ct)
    with pytest.raises(TypeError):
        ctx.decrypt_int(sk, packed, 2)
    with pytest.raises(ValueError):
        ctx.decrypt(psk2, packed)                                 # a k = 2 packing key for a k = 1 packed array
    other = nufhe_b200.LweSampleArray(nufhe_b200.lwe.LweParams(500, 1e-3, 1e-2), ct.a, ct.b, ct.current_variances)
    with pytest.raises(ValueError):
        packing.pack(ctx.thread, pk, other)
    assert (ctx.decrypt(sk, ct) == [True, False]).all()          # the LWE path is as before


def test_empty_batch(keys):
    ctx, sk, psk, pk = keys
    ct = ctx.encrypt(sk, numpy.zeros((0, 3), bool))
    packed = packing.pack(ctx.thread, pk, ct)
    assert tuple(packed.data.shape) == (0, 2, 1024)
    assert ctx.decrypt(psk, packed).shape == (0, 3)
