"""Compact public-key encryption on the CPU: the rounding and extraction functions of csrc/compact_layout.cuh (through
the host emulator) against the NumPy restatement (compact_ref.py), and the Python layer (nufhe_b200/compact.py) on the
oracle-backed engine double: draw order and byte-identity of the other keys, the phase of the key, encrypt / expand /
decrypt round trips bit-exact against the restatement, pickles, argument errors, and the noise figures of DESIGN.md
section 16."""
import copy
import ctypes
import io
import os

import numpy
import pytest

import nufhe_b200
from nufhe_b200 import compact
from nufhe_b200.compressed import draw_seed
from nufhe_b200.lut import encode_int
from nufhe_b200.api_low_level import bool_to_t32
from nufhe_b200.random_numbers import DeterministicRNG
from chacha_ref import seeded_uniform
from fake_engine import _np, _t
from oracle import oracle as O
from test_host_pack import PackingFakeEngine
import compact_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 1024
P = 0xffffffff00000001
SIGMA = 9e-9 * (2 / numpy.pi)**0.5
BOUNDARY = [0, 2**15 - 1, 2**15, 0x7fff8000, 0xffff8000, -1, -2**31]


@pytest.fixture(scope='module')
def emul():
    path = os.path.join(ROOT, 'nufhe_b200', 'csrc', 'libnb_host_emul.so')
    if not os.path.exists(path):
        import __graft_entry__ as g
        g.build()
    lib = ctypes.CDLL(path)
    lib.emul_compact_coeff.argtypes = [ctypes.c_void_p] * 5 + [ctypes.c_size_t, ctypes.c_void_p]
    lib.emul_compact_coeff.restype = None
    lib.emul_compact_extract.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p]
    lib.emul_compact_extract.restype = None
    return lib


def _coeffs(emul, product, noise, body, occupied, mu):
    arrs = [numpy.ascontiguousarray(compact_ref.u32(x).astype(numpy.uint32)) for x in (product, noise, mu)]
    flags = [numpy.ascontiguousarray(numpy.asarray(f, numpy.uint8)) for f in (body, occupied)]
    out = numpy.empty(arrs[0].size, numpy.uint16)
    emul.emul_compact_coeff(arrs[0].ctypes.data, arrs[1].ctypes.data, flags[0].ctypes.data, flags[1].ctypes.data,
                            arrs[2].ctypes.data, out.size, out.ctypes.data)
    return out


def test_header_rounding(emul):
    x = numpy.array(BOUNDARY, numpy.int64)
    zero = numpy.zeros_like(x)
    ones = numpy.ones(x.size, numpy.uint8)
    got = _coeffs(emul, x, zero, ones * 0, ones * 0, zero)                     # mask coefficients
    assert list(got) == [0, 0, 1, 0x8000, 0, 0, 0x8000]
    assert (got == compact_ref.round16(x)).all()
    # the sum is taken mod 2^32 before the rounding; the message counts on an occupied body slot only
    rng = numpy.random.RandomState(1)
    prod, noise, mu = (rng.randint(-2**31, 2**31, size=4096, dtype=numpy.int64) for _ in range(3))
    body, occ = rng.randint(0, 2, (2, 4096)).astype(numpy.uint8)
    got = _coeffs(emul, prod, noise, body, occ, mu)
    want = compact_ref.round16(prod + noise + numpy.where(body & occ, mu, 0))
    want[(body == 1) & (occ == 0)] = 0
    assert (got == want).all()


@pytest.mark.parametrize('k', [1, 2])
def test_header_extraction(emul, k):
    rng = numpy.random.RandomState(k)
    data = rng.randint(0, 2**16, size=(1, k + 1, N)).astype(numpy.uint16)
    data[0, :, :4] = [0, 0x7fff, 0x8000, 0xffff]
    data[0, :, -2:] = [0x8000, 0xffff]
    want_a, want_b = compact_ref.extract(data, N)
    x = compact_ref.unround16(data).astype(numpy.int64)
    for p in (0, 1, N - 1):
        a = numpy.empty(k * N, numpy.int32)
        b = numpy.empty(1, numpy.int32)
        emul.emul_compact_extract(data.ctypes.data, k, p, a.ctypes.data, b.ctypes.data)
        assert (a == want_a[p]).all() and b[0] == want_b[p] == compact_ref.i32(x[0, k, p])
        for u in range(k):
            for j in sorted({0, p, p + 1, N - 1} - {N}):
                want = x[0, u, p - j] if j <= p else -x[0, u, N + p - j]
                assert a[u * N + j] == compact_ref.i32(want), (p, u, j)
    # p = 0 is tlwe_extract_lwe_samples' convention
    a0 = numpy.empty(k * N, numpy.int32)
    emul.emul_compact_extract(data.ctypes.data, k, 0, a0.ctypes.data, b.ctypes.data)
    ref = numpy.concatenate([[x[0, u, 0]] + list(-x[0, u, :0:-1]) for u in range(k)])
    assert (a0 == compact_ref.i32(ref)).all()


def test_exactness_bound_and_noise_figures():
    """Every coefficient of A_u r is at most N 2^31 < p / 2 in magnitude, so the NTT chain gives it exactly mod 2^32;
    the DESIGN.md section 16 noise figures for k = 1."""
    assert N * 2**31 < P // 2
    for k in (1, 2):
        params = nufhe_b200.NuFHEParameters(tlwe_mask_size=k)
        assert numpy.allclose(compact.noise_terms(params), compact_ref.noise_terms(params), rtol=1e-12, atol=0)
    fresh, mask, body, ks = compact.noise_terms(nufhe_b200.NuFHEParameters())
    assert abs(fresh - 5.3e-14) < 0.05e-14 and abs(mask - 9.9e-9) < 0.05e-9 and abs(body - 1.9e-11) < 0.05e-11
    assert abs(ks - 3.64e-6) < 0.01e-6
    total = fresh + mask + body + ks
    assert abs(total - 3.65e-6) < 0.01e-6 and total < 4.86e-6 < 1.28e-5
    assert compact.groups_per_pass(nufhe_b200.NuFHEParameters()) == 16


# ---------------------------------------------------------------- the Python layer on the engine double

class CompactFakeEngine(PackingFakeEngine):
    """PackingFakeEngine with Engine.compact_finish / compact_extract (nb_compact_finish, nb_compact_extract) restated
    with NumPy."""

    def compact_finish(self, c, e1, e2, mus):
        self._count('compact_finish')
        return _t(compact_ref.finish(compact_ref.u32(_np(c)), _np(e1), _np(e2), _np(mus)))

    def compact_extract(self, data, rows):
        self._count('compact_extract')
        a, b = compact_ref.extract(_np(data), rows)
        return _t(a), _t(b)


def _context(seed):
    return nufhe_b200.Context(rng=DeterministicRNG(seed), thread=CompactFakeEngine())


def _keys(seed, k):
    ctx = _context(seed)
    sk = ctx.make_secret_key(tlwe_mask_size=k)
    ck, cpk = ctx.make_cloud_key(sk, compact_public_key=True)
    return ctx, sk, ck, cpk, ctx.make_virtual_machine(ck)


@pytest.fixture(scope='module')
def keys():
    return _keys(81, 1)


@pytest.fixture(scope='module')
def keys2():
    return _keys(82, 2)


def _glwe_key(seed, k):
    replay = DeterministicRNG(seed)
    replay.uniform_bool((500,))
    return replay.uniform_bool((k, N))                   # the TGSW key's TLWE key, drawn first by make_cloud_key


def _key_polys(cpk):
    k = cpk.params.tgsw_params.tlwe_params.mask_size
    return numpy.concatenate([seeded_uniform(cpk.seed, compact.NONCE_COMPACT_KEY, (k, N)), _np(cpk.b)[None]])


@pytest.mark.parametrize('k', [1, 2])
def test_key_draw_order_and_phase(keys, keys2, k):
    ctx, sk, ck, cpk, vm = keys if k == 1 else keys2
    seed = 81 if k == 1 else 82
    ctx2 = _context(seed)
    sk2 = ctx2.make_secret_key(tlwe_mask_size=k)
    ck2 = ctx2.make_cloud_key(sk2)
    assert ck2.dumps() == ck.dumps()
    assert (draw_seed(ctx2.rng) == cpk.seed).all()                  # the seed, then E, after every other key
    E = O.double_to_t32(ctx2.rng.gauss((N,), SIGMA)).astype(numpy.int64)
    assert isinstance(cpk, nufhe_b200.NuFHECompactPublicKey) and tuple(cpk.b.shape) == (N,)
    polys = _key_polys(cpk).astype(numpy.int64)
    S = _glwe_key(seed, k)
    err = polys[k].copy()
    for u in range(k):
        err -= polys[u] @ compact_ref.negacyclic_matrix(S[u])
    err = compact_ref.i32(err).astype(numpy.int64)
    assert (err == E).all()                                         # B - A.S = E exactly
    assert numpy.abs(err).max() < 8 * SIGMA * 2**32


def test_other_keys_are_byte_identical():
    """Cloud, tree and index keys with and without the flag, plain and compressed."""
    for compressed in (False, True):
        c1, c2 = _context(83), _context(83)
        s1, s2 = c1.make_secret_key(), c2.make_secret_key()
        with_flag = c1.make_cloud_key(s1, compressed=compressed, tree_key=True, index_key=True, compact_public_key=True)
        without = c2.make_cloud_key(s2, compressed=compressed, tree_key=True, index_key=True)
        assert len(with_flag) == 4 and isinstance(with_flag[3], nufhe_b200.NuFHECompactPublicKey)
        for x, y in zip(with_flag[:3], without):
            assert x.dumps() == y.dumps()
        assert (draw_seed(c2.rng) == with_flag[3].seed).all()


def _encrypt_and_replay(ctx, cpk, message, bits=None):
    """ctx.encrypt (bits is None) or ctx.encrypt_int, and the restatement's data from a replay of the same draws."""
    k = cpk.params.tgsw_params.tlwe_params.mask_size
    replay = copy.deepcopy(ctx.rng)
    ct = ctx.encrypt(cpk, message) if bits is None else ctx.encrypt_int(cpk, message, bits)
    mus = bool_to_t32(message) if bits is None else encode_int(numpy.asarray(message), bits)
    G = -(-mus.size // N)
    r_seed = draw_seed(replay)
    e1 = O.double_to_t32(replay.gauss((G, k, N), SIGMA))
    e2 = O.double_to_t32(replay.gauss((G, N), SIGMA))
    words = seeded_uniform(r_seed, compact.NONCE_COMPACT_RANDOMNESS, (G, N // 32))
    return ct, compact_ref.encrypt(_key_polys(cpk), words, e1, e2, mus.reshape(-1))


def _check(ctx, sk, ck, cpk, vm, message, bits=None):
    ct, want = _encrypt_and_replay(ctx, cpk, message, bits)
    assert isinstance(ct, nufhe_b200.CompactLweSampleArray) and ct.shape == numpy.shape(message)
    assert (_np(ct.data) == want).all()
    out = vm.expand(ct)
    ks = tuple(_np(x) for x in ck.keyswitch_key.device_arrays())
    ra, rb, rcv = compact_ref.expand(want, ct.size, ks)
    assert isinstance(out, nufhe_b200.LweSampleArray) and out.shape == ct.shape
    assert (_np(out.a).reshape(ra.shape) == ra).all() and (_np(out.b).reshape(-1) == rb).all()
    est = sum(compact.noise_terms(ck.params)[:3])
    assert numpy.allclose(_np(out.current_variances).reshape(-1), rcv + est, rtol=1e-6)
    got = ctx.decrypt(sk, out) if bits is None else ctx.decrypt_int(sk, out, bits)
    assert got.shape == numpy.shape(message) and (got == message).all()


@pytest.mark.parametrize('k', [1, 2])
@pytest.mark.parametrize('shape', [(1,), (1023,), (1024,), (1025,), (3, 700)])
def test_encrypt_expand_decrypt_bits(keys, keys2, k, shape):
    ctx, sk, ck, cpk, vm = keys if k == 1 else keys2
    bits = numpy.random.RandomState(sum(shape) + k).randint(0, 2, size=shape).astype(bool)
    _check(ctx, sk, ck, cpk, vm, bits)


@pytest.mark.parametrize('k', [1, 2])
@pytest.mark.parametrize('shape', [(1,), (1025,), (3, 700)])
def test_encrypt_expand_decrypt_2bit_integers(keys, keys2, k, shape):
    ctx, sk, ck, cpk, vm = keys if k == 1 else keys2
    values = numpy.random.RandomState(sum(shape) + 10 * k).randint(0, 4, size=shape)
    _check(ctx, sk, ck, cpk, vm, values, bits=2)


def test_expansion_in_passes(keys, monkeypatch):
    """A batch across a pass boundary gives the same samples as one pass."""
    ctx, sk, ck, cpk, vm = keys
    bits = numpy.random.RandomState(9).randint(0, 2, size=2500).astype(bool)
    ct = ctx.encrypt(cpk, bits)
    whole = vm.expand(ct)
    monkeypatch.setattr(compact, 'PASS_BYTES', 4 * N * N)           # one group per pass
    assert compact.groups_per_pass(ck.params) == 1
    calls = ctx.thread.calls.get('compact_extract', 0)
    parts = vm.expand(ct)
    assert ctx.thread.calls['compact_extract'] - calls == 3
    assert (_np(parts.a) == _np(whole.a)).all() and (_np(parts.b) == _np(whole.b)).all()
    assert (_np(parts.current_variances) == _np(whole.current_variances)).all()
    assert (ctx.decrypt(sk, parts) == bits).all()


def test_pickles_and_sizes(keys):
    ctx, sk, ck, cpk, vm = keys
    s = cpk.dumps()
    assert 4096 < len(s) < 5400               # the 4 KB body, the seed and the params
    assert ctx.load_compact_public_key(s) == cpk and ctx.load_compact_public_key(io.BytesIO(s)) == cpk
    bits = numpy.arange(1030) % 3 == 0
    ct = ctx.encrypt(ctx.load_compact_public_key(s), bits)
    c = ct.dumps()
    assert len(c) <= 2 * 2 * N * 2 + 1024
    back = ctx.load_compact_ciphertext(c)
    assert back == ct and ctx.load_compact_ciphertext(io.BytesIO(c)) == ct
    assert (ctx.decrypt(sk, vm.expand(back)) == bits).all()
    loaders = (ctx.load_compact_public_key, ctx.load_compact_ciphertext)
    others = (sk.dumps(), ctx.encrypt(sk, [True], compressed=True).dumps(), b'junk')
    for i, load in enumerate(loaders):
        for j, wrong in enumerate((s, c) + others):
            if i != j:
                with pytest.raises(ValueError):
                    load(wrong)
    with pytest.raises(ValueError):                                 # a truncated ciphertext
        ctx.load_compact_ciphertext(c[:-100])


def test_argument_errors(keys, keys2):
    ctx, sk, ck, cpk, vm = keys
    ctx2, sk2, ck2, cpk2, vm2 = keys2
    with pytest.raises(ValueError):
        ctx.encrypt(cpk, [True], compressed=True)
    with pytest.raises(ValueError):
        ctx.encrypt_int(cpk, [1], 2, compressed=True)
    with pytest.raises(ValueError):
        vm.expand(ctx2.encrypt(cpk2, [True, False]))                # k = 2 ciphertexts on a k = 1 machine
    with pytest.raises(TypeError):
        vm.expand(ctx.encrypt(sk, [True]))
    with pytest.raises(TypeError):
        vm.expand(ctx.encrypt(sk, [True], compressed=True))
    with pytest.raises(ValueError):
        nufhe_b200.CompactLweSampleArray(ck.params, (1025,), ctx.encrypt(cpk, [True]).data)


def test_empty_batch(keys):
    ctx, sk, ck, cpk, vm = keys
    ct = ctx.encrypt(cpk, numpy.zeros((0, 3), bool))
    assert tuple(ct.data.shape) == (0, 2, N)
    out = vm.expand(ct)
    assert out.shape == (0, 3) and ctx.decrypt(sk, out).shape == (0, 3)
