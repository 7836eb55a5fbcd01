"""Public-key encryption on the CPU: the kernel's tile loop and index arithmetic (csrc/plane_gemm.cuh, pk_layout.cuh,
through the host emulator's scalar model of the m16n8k32 u8 MMA) against an independent NumPy restatement (pk_ref.py), and the Python
layer (nufhe_b200/public_key.py) on an oracle-backed engine double: draw order, the phase error of every ciphertext,
variances, decryption, serialization, a gate, and the noise bound of DESIGN.md section 11."""
import ctypes
import io
import os

import numpy
import pytest

import nufhe_b200
from nufhe_b200 import lut
from nufhe_b200.public_key import NONCE_ENCRYPTION_RANDOMNESS, public_key_size
from nufhe_b200.random_numbers import DeterministicRNG
from chacha_ref import seeded_uniform
from fake_engine import FakeEngine, _np, _t
from oracle import oracle as O
import pk_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIGMA = 2**-15 * (2 / numpy.pi)**0.5


@pytest.fixture(scope='module')
def emul():
    path = os.path.join(ROOT, 'nufhe_b200', 'csrc', 'libnb_host_emul.so')
    if not os.path.exists(path):
        import __graft_entry__ as g
        g.build()
    lib = ctypes.CDLL(path)
    lib.emul_pk_encrypt.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t,
                                    ctypes.c_size_t, ctypes.c_void_p, ctypes.c_float, ctypes.c_void_p,
                                    ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t]
    lib.emul_pk_encrypt.restype = None
    return lib


def _emul_encrypt(lib, masks, pk_b, r_words, mus, variance):
    masks, pk_b = numpy.ascontiguousarray(masks, numpy.int32), numpy.ascontiguousarray(pk_b, numpy.int32)
    r_words, mus = numpy.ascontiguousarray(r_words, numpy.int32), numpy.ascontiguousarray(mus, numpy.int32)
    m, n = masks.shape
    B = mus.size
    a, b, cv = numpy.empty((B, n), numpy.int32), numpy.empty(B, numpy.int32), numpy.empty(B, numpy.float32)
    lib.emul_pk_encrypt(r_words.ctypes.data, masks.ctypes.data, pk_b.ctypes.data, m, n, mus.ctypes.data,
                        ctypes.c_float(variance), a.ctypes.data, b.ctypes.data, cv.ctypes.data, B)
    return a, b, cv


def _i32(rng, shape):
    return rng.randint(-2**31, 2**31, size=shape, dtype=numpy.int64).astype(numpy.int32)


def _case(kind, m, n, B, seed):
    """(masks, b, R words, mus) of a generated key or an adversarial one."""
    rng = numpy.random.RandomState(seed)
    masks, pk_b = _i32(rng, (m, n)), _i32(rng, m)
    words = _i32(rng, (B, m // 32))
    mus = _i32(rng, B)
    if kind == 'max':                       # every product and sum as large as it gets
        masks[:] = -1
        pk_b[:] = -2**31
        words[:] = -1
    elif kind == 'first_bit':
        words[:] = 0
        words[:, 0] = 1
    elif kind == 'last_bit':
        words[:] = 0
        words[:, -1] = -2**31
    return masks, pk_b, words, mus


def _check(lib, masks, pk_b, words, mus):
    var = float(numpy.float32(SIGMA**2))
    got = _emul_encrypt(lib, masks, pk_b, words, mus, var)
    want = pk_ref.encrypt(masks, pk_b, words, mus, var)
    for g, w in zip(got, want):
        assert g.shape == w.shape and (g.view(numpy.uint32) == w.view(numpy.uint32)).all()


@pytest.mark.parametrize('B', [1, 15, 16, 17, 129])
@pytest.mark.parametrize('m', [32, 64, 16384])
def test_emulated_kernel_matches_the_restatement(emul, m, B):
    _check(emul, *_case('random', m, 500, B, m + B))


@pytest.mark.parametrize('kind', ['max', 'first_bit', 'last_bit'])
@pytest.mark.parametrize('m', [32, 64, 16384])
def test_emulated_kernel_on_adversarial_keys(emul, m, kind):
    _check(emul, *_case(kind, m, 500, 17, m))


@pytest.mark.parametrize('n', [1, 6, 7, 13])
def test_emulated_kernel_padding_columns(emul, n):
    """n + 2 columns padded to a multiple of 8: b and the ones column fall in different lanes and tiles."""
    _check(emul, *_case('random', 96, n, 70, n))


# ---------------------------------------------------------------- the Python layer on the engine double

class PublicKeyFakeEngine(FakeEngine):
    """FakeEngine with Engine.seeded_uniform from the NumPy keystream and Engine.pk_prepare / public_encrypt from the
    NumPy restatement (the 'planes' are the key's arrays themselves)."""

    def seeded_uniform(self, seed, nonce, shape, first=0):
        self._count('seeded_uniform')
        return _t(seeded_uniform(seed, nonce, shape, first))

    def pk_prepare(self, a, b):
        self._count('pk_prepare')
        return _np(a).copy(), _np(b).copy()

    def public_encrypt(self, r_words, planes, m, n, mus, row_variance):
        self._count('public_encrypt')
        masks, pk_b = planes
        assert masks.shape == (m, n)
        a, b, cv = pk_ref.encrypt(masks, pk_b, _np(r_words), _np(mus), row_variance)
        return _t(a), _t(b), _t(cv)


def _context(seed):
    return nufhe_b200.Context(rng=DeterministicRNG(seed), thread=PublicKeyFakeEngine())


def _wrap(x):
    return (numpy.asarray(x, numpy.int64) & 0xffffffff).astype(numpy.uint32).view(numpy.int32)


@pytest.fixture(scope='module')
def keys():
    """Context, secret key, public key, and the replayed RNG after key generation with the key's noises e."""
    ctx = _context(51)
    sk = ctx.make_secret_key()
    pk = ctx.make_public_key(sk)
    m = public_key_size(sk.params)
    replay = DeterministicRNG(51)
    replay.uniform_bool((500,))
    assert (pk.seed.view(numpy.int32) == replay.uniform_torus32((8,))).all()
    e = O.double_to_t32(replay.gauss((m,), sk.params.in_out_params.min_noise))
    return ctx, sk, pk, e


def test_public_key_generation(keys):
    ctx, sk, pk, e = keys
    assert pk.size == 16384 and tuple(pk.b.shape) == (16384,)
    assert pk.variance == float(numpy.float32(SIGMA**2))
    masks = seeded_uniform(pk.seed, 0, (16384, 500))
    dot = (masks.astype(numpy.int64) * _np(sk.lwe_key.key).astype(numpy.int64)).sum(-1)
    assert (_np(pk.b) == _wrap(dot + e)).all()                    # encryptions of 0 with the noises drawn
    assert (_np(pk.masks(ctx.thread)) == masks).all()


def _phase(sk, ct):
    key = _np(sk.lwe_key.key).astype(numpy.int64)
    return _wrap(_np(ct.b).astype(numpy.int64) - (_np(ct.a).astype(numpy.int64) * key).sum(-1))


def test_encryption_draws_one_seed_and_has_the_phase_error_of_its_rows():
    ctx = _context(52)
    sk = ctx.make_secret_key()
    pk = ctx.make_public_key(sk)
    m = pk.size
    replay = DeterministicRNG(52)
    replay.uniform_bool((500,))
    replay.uniform_torus32((8,))
    e = O.double_to_t32(replay.gauss((m,), sk.params.in_out_params.min_noise)).astype(numpy.int64)
    bits = numpy.random.RandomState(2).randint(0, 2, size=(3, 5)).astype(bool)
    calls = dict(ctx.thread.calls)
    ct = ctx.encrypt(pk, bits)
    assert isinstance(ct, nufhe_b200.LweSampleArray) and tuple(ct.b.shape) == (3, 5) and tuple(ct.a.shape) == (3, 5, 500)
    assert ctx.thread.calls['public_encrypt'] == calls.get('public_encrypt', 0) + 1
    # the call drew 8 words (the R seed) and nothing else
    r_seed = replay.uniform_torus32((8,)).view(numpy.uint32)
    assert (ctx.rng.uniform_torus32((16,)) == replay.uniform_torus32((16,))).all()
    R = pk_ref.r_bits(seeded_uniform(r_seed, NONCE_ENCRYPTION_RANDOMNESS, (15, m // 32)), m).astype(numpy.int64)
    mus = nufhe_b200.api_low_level.bool_to_t32(bits).reshape(-1).astype(numpy.int64)
    # phase - mu = sum_i r_i e_i exactly (mod 2^32), with e the key's noises
    assert (_phase(sk, ct).reshape(-1) == _wrap(mus + R @ e)).all()
    pop = R.sum(1)
    assert 0 < pop.min() and pop.max() < m
    assert (_np(ct.current_variances).reshape(-1) == pop.astype(numpy.float32) * numpy.float32(SIGMA**2)).all()
    assert (ctx.decrypt(sk, ct) == bits).all()


def test_two_encryptions_use_different_r(keys):
    ctx, sk, pk, e = keys
    bits = numpy.ones(4, bool)
    c1, c2 = ctx.encrypt(pk, bits), ctx.encrypt(pk, bits)
    assert not (_np(c1.a) == _np(c2.a)).all(axis=-1).any()
    assert (ctx.decrypt(sk, c1) == bits).all() and (ctx.decrypt(sk, c2) == bits).all()


def test_encrypt_int_and_decryption(keys):
    ctx, sk, pk, e = keys
    for bits in (1, 2, 3):
        values = numpy.arange(24) % (2**bits)
        assert (ctx.decrypt_int(sk, ctx.encrypt_int(pk, values, bits), bits) == values).all()
    one = ctx.encrypt(pk, True)
    assert tuple(one.b.shape) == () and ctx.decrypt(sk, one)


def test_public_key_serialization(keys):
    ctx, sk, pk, e = keys
    s = pk.dumps()
    back = ctx.load_public_key(s)
    assert back == pk and ctx.load_public_key(io.BytesIO(s)) == pk
    assert len(s) <= 70e3
    assert (ctx.decrypt(sk, ctx.encrypt(back, [True, False, True])) == [True, False, True]).all()
    for wrong in (ctx.encrypt(sk, [True], compressed=True).dumps(), sk.dumps(), b'not a pickle'):
        with pytest.raises(ValueError):
            ctx.load_public_key(wrong)
    with pytest.raises(ValueError):
        nufhe_b200.CompressedLweSampleArray.loads(s, ctx.thread)


def test_compressed_public_encryption_raises(keys):
    ctx, sk, pk, e = keys
    with pytest.raises(ValueError):
        ctx.encrypt(pk, [True], compressed=True)
    with pytest.raises(ValueError):
        ctx.encrypt_int(pk, [1], 2, compressed=True)


def test_gate_nand_on_public_key_ciphertexts():
    ctx = _context(53)
    sk = ctx.make_secret_key()
    pk = ctx.make_public_key(sk)
    ck = ctx.make_cloud_key(sk)
    vm = ctx.make_virtual_machine(ck)
    x = numpy.arange(8) % 2 == 1
    y = numpy.arange(8) // 2 % 2 == 1
    cx, cy = ctx.encrypt(pk, x), ctx.encrypt(pk, y)
    r = vm.gate_nand(cx, cy)
    assert (ctx.decrypt(sk, r) == ~(x & y)).all()
    ks = ck.keyswitch_key.device_arrays()
    want = O.gate_binary('nand', (_np(cx.a), _np(cx.b)), (_np(cy.a), _np(cy.b)),
                         _np(ck.bootstrap_key.tgsw.samples.a.coeffs, True), tuple(_np(v) for v in ks))
    assert (_np(r.a) == want[0]).all() and (_np(r.b) == want[1]).all()


@pytest.mark.parametrize('k', [1, 2])
def test_public_key_noise_is_below_a_lut_output(k):
    """m sigma^2 (every bit of R set) is below the variance of one LUT output before the mod-switch, the input noise
    lut.check_noise and the gates already allow for.  sigma(x + y)^2 - sigma(x)^2 is exactly that variance."""
    params = nufhe_b200.NuFHEParameters(tlwe_mask_size=k)
    io_params = params.in_out_params
    assert io_params.min_noise == SIGMA
    m = public_key_size(params)
    assert m == 16384 and m >= (io_params.size + 1) * 32 + 256

    def est(shift):
        return lut._sigma_estimate(io_params, params.tgsw_params, params.ks_decomp_length, params.ks_log2_base, 0,
                                   shift)**2
    lut_output = est(0) - est(None)
    assert m * SIGMA**2 < lut_output
    assert abs(m * SIGMA**2 - 9.71e-6) < 0.01e-6 and abs(m / 2 * SIGMA**2 - 4.86e-6) < 0.01e-6
