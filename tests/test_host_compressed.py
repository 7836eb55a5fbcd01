"""Compressed keys and ciphertexts on the CPU: the ChaCha20 keystream of the seeded masks (the NumPy reference in
chacha_ref.py and the kernel's own block function, csrc/chacha.cuh through the host emulator) against RFC 8439 and
against each other, and the Python layer (nufhe_b200/compressed.py) on an oracle-backed engine double: draw order,
serialization, decryption, gates on a decompressed cloud key and the phase of every decompressed key row."""
import ctypes
import os

import numpy
import pytest
import torch

import nufhe_b200
from nufhe_b200 import compressed as C
from nufhe_b200.random_numbers import DeterministicRNG
from chacha_ref import chacha20_blocks, chacha20_words, seeded_uniform
from fake_engine import FakeEngine, _np, _t
from oracle import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 1024

RFC_KEY = numpy.frombuffer(bytes(range(32)), '<u4')
RFC_BLOCK = ('10f1e7e4d13b5915500fdd1fa32071c4c7d1f4c733c068030422aa9ac3d46c4e'
             'd2826446079faa0914c2d705d98b02a2b5129cd1de164eb9cbd083e8a2503c4e')
ZERO_BLOCK0 = ('76b8e0ada0f13d90405d6ae55386bd28bdd219b8a08ded1aa836efcc8b770dc7'
               'da41597c5157488d7724e03fb8d84a376a43b8f41518a11cc387b669b2ee6586')
ZERO_BLOCK1 = ('9f07e7be5551387a98ba977c732d080dcb0f29a048e3656912c6533e32ee7aed'
               '29b721769ce64e43d57133b074d839d531ed1f28510afb45ace10a1f4b794d6f')
# RFC 8439 section 2.3.2: state words 12-15 = 1, 0x09000000, 0x4a000000, 0 -> counter, nonce of the 64-bit layout
RFC_COUNTER, RFC_NONCE = 1 | (0x09000000 << 32), 0x4a000000


@pytest.fixture(scope='module')
def emul():
    path = os.path.join(ROOT, 'nufhe_b200', 'csrc', 'libnb_host_emul.so')
    if not os.path.exists(path):
        import __graft_entry__ as g
        g.build()
    lib = ctypes.CDLL(path)
    lib.emul_chacha_block.argtypes = [ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_void_p]
    lib.emul_chacha_block.restype = None
    return lib


def _emul_block(lib, seed, counter, nonce):
    seed = numpy.ascontiguousarray(numpy.asarray(seed).astype(numpy.int64).astype(numpy.uint32))
    out = numpy.empty(16, numpy.uint32)
    lib.emul_chacha_block(seed.ctypes.data, ctypes.c_uint64(counter), ctypes.c_uint64(nonce), out.ctypes.data)
    return out


def _hex(words):
    return numpy.asarray(words).astype('<u4').tobytes().hex()


# ---------------------------------------------------------------- the keystream

def test_reference_matches_rfc8439():
    assert _hex(chacha20_blocks(RFC_KEY, RFC_NONCE, [RFC_COUNTER])[0]) == RFC_BLOCK
    zero = numpy.zeros(8, numpy.uint32)
    blocks = chacha20_blocks(zero, 0, [0, 1])
    assert _hex(blocks[0]) == ZERO_BLOCK0
    assert _hex(blocks[1]) == ZERO_BLOCK1
    assert _hex(chacha20_words(zero, 0, 0, 32).view(numpy.uint32)) == ZERO_BLOCK0 + ZERO_BLOCK1


def test_kernel_block_function_matches_rfc8439(emul):
    assert _hex(_emul_block(emul, RFC_KEY, RFC_COUNTER, RFC_NONCE)) == RFC_BLOCK
    zero = numpy.zeros(8, numpy.uint32)
    assert _hex(_emul_block(emul, zero, 0, 0)) == ZERO_BLOCK0
    assert _hex(_emul_block(emul, zero, 1, 0)) == ZERO_BLOCK1


def _cryptography_stream(seed, nonce, first_block, blocks):
    ciphers = pytest.importorskip('cryptography.hazmat.primitives.ciphers')
    # its 16-byte nonce is state words 12-15: the 64-bit block counter, then our 64-bit nonce
    iv = int(first_block).to_bytes(8, 'little') + int(nonce).to_bytes(8, 'little')
    key = numpy.asarray(seed).astype('<u4').tobytes()
    enc = ciphers.Cipher(ciphers.algorithms.ChaCha20(key, iv), mode=None).encryptor()
    return numpy.frombuffer(enc.update(bytes(64 * blocks)), '<u4').view(numpy.int32)


@pytest.mark.parametrize('first_block, blocks', [(0, 5), (2**32 - 1, 3), (2**32 - 2, 4), (12345678901, 2)])
def test_reference_matches_cryptography(first_block, blocks):
    rng = numpy.random.RandomState(first_block % 1000)
    seed = rng.randint(0, 2**32, size=8, dtype=numpy.uint64).astype(numpy.uint32)
    nonce = int(rng.randint(0, 2**62))
    want = _cryptography_stream(seed, nonce, first_block, blocks)
    got = chacha20_words(seed, nonce, 16 * first_block, 16 * blocks)
    assert (got == want).all()
    # a range that starts and ends mid-block
    assert (chacha20_words(seed, nonce, 16 * first_block + 5, 16 * blocks - 9) == want[5:-4]).all()


def test_kernel_block_function_matches_reference(emul):
    rng = numpy.random.RandomState(8439)
    counters = [0, 1, 2**32 - 1, 2**32, 2**33 + 7, 2**63, 2**64 - 1] + list(rng.randint(0, 2**63, size=20))
    for i, counter in enumerate(counters):
        seed = rng.randint(0, 2**32, size=8, dtype=numpy.uint64).astype(numpy.uint32)
        nonce = [0, 1, 2, 2**64 - 1][i % 4] if i < 8 else int(rng.randint(0, 2**63)) * 2 + 1
        want = chacha20_blocks(seed, nonce, [counter])[0]
        assert (_emul_block(emul, seed, int(counter), nonce) == want).all(), (counter, nonce)


def test_words_carry_into_counter_high_word():
    seed = numpy.arange(8, dtype=numpy.uint32) * 0x01010101
    first = 16 * (2**32 - 1) + 3                      # 13 words of block 2^32 - 1, then block 2^32
    got = chacha20_words(seed, 7, first, 40)
    b = chacha20_blocks(seed, 7, [2**32 - 1, 2**32, 2**32 + 1]).reshape(-1).view(numpy.int32)
    assert (got == b[3:43]).all()
    # block 2^32 is not block 0: the carry reaches state word 13
    assert not (chacha20_blocks(seed, 7, [2**32])[0] == chacha20_blocks(seed, 7, [0])[0]).all()


# ---------------------------------------------------------------- the Python layer on the engine double

class SeededFakeEngine(FakeEngine):
    """FakeEngine with Engine.seeded_uniform from the NumPy keystream."""

    def seeded_uniform(self, seed, nonce, shape, first=0):
        self._count('seeded_uniform')
        return _t(seeded_uniform(seed, nonce, shape, first))


def _context(seed):
    return nufhe_b200.Context(rng=DeterministicRNG(seed), thread=SeededFakeEngine())


def _wrap(x):
    return (numpy.asarray(x, numpy.int64) & 0xffffffff).astype(numpy.uint32).view(numpy.int32)


def test_compressed_encrypt_draw_order_and_decryption():
    ctx = _context(31)
    sk = ctx.make_secret_key()
    bits = numpy.random.RandomState(1).randint(0, 2, size=(3, 7)).astype(bool)
    ct = ctx.encrypt(sk, bits, compressed=True)
    assert isinstance(ct, nufhe_b200.CompressedLweSampleArray) and ct.shape == (3, 7)
    # the seed is the next 8 Torus32 draws, then come the Gaussian noises of b, as in lwe_encrypt
    replay = DeterministicRNG(31)
    replay.uniform_bool((500,))
    assert (ct.seed.view(numpy.int32) == replay.uniform_torus32((8,))).all()
    noise = sk.params.in_out_params.min_noise
    e = O.double_to_t32(replay.gauss(bits.shape, noise))
    a = seeded_uniform(ct.seed, C.NONCE_CIPHERTEXT, bits.shape + (500,))
    dot = (a.astype(numpy.int64) * _np(sk.lwe_key.key).astype(numpy.int64)).sum(-1)
    mus = nufhe_b200.api_low_level.bool_to_t32(bits).astype(numpy.int64)
    assert (_np(ct.b) == _wrap(mus + e + dot)).all()

    full = ct.decompress(ctx.thread)
    assert (_np(full.a) == a).all() and (_np(full.b) == _np(ct.b)).all()
    assert (_np(full.current_variances) == numpy.float32(noise**2)).all()
    assert (ctx.decrypt(sk, full) == bits).all()
    # the ordinary path still draws the mask from the RNG
    assert isinstance(ctx.encrypt(sk, bits), nufhe_b200.LweSampleArray)


def test_compressed_encrypt_int():
    ctx = _context(32)
    sk = ctx.make_secret_key()
    for bits in (1, 2):
        values = numpy.arange(40) % (2**bits)
        ct = ctx.encrypt_int(sk, values, bits, compressed=True)
        assert (ctx.decrypt_int(sk, ct.decompress(ctx.thread), bits) == values).all()


def test_compressed_ciphertext_serialization():
    ctx = _context(33)
    sk = ctx.make_secret_key()
    bits = numpy.array([[1, 0, 1], [0, 0, 1]], bool)
    ct = ctx.encrypt(sk, bits, compressed=True)
    s = ct.dumps()
    back = ctx.load_compressed_ciphertext(s)
    assert back == ct
    assert back.decompress(ctx.thread) == ct.decompress(ctx.thread)
    import io
    assert ctx.load_compressed_ciphertext(io.BytesIO(s)) == ct
    assert len(s) < 1000
    # a scalar message
    one = ctx.encrypt(sk, True, compressed=True)
    assert one.shape == () and ctx.decrypt(sk, ctx.load_compressed_ciphertext(one.dumps()).decompress(ctx.thread))
    # wrong kinds of pickle
    with pytest.raises(ValueError):
        ctx.load_compressed_ciphertext(ctx.encrypt(sk, bits).dumps())
    with pytest.raises(ValueError):
        nufhe_b200.CompressedCloudKey.loads(s, ctx.thread)
    with pytest.raises(ValueError):
        ctx.load_compressed_ciphertext(b'not a pickle')


def test_two_contexts_seeded_alike_give_identical_dumps():
    dumps = []
    for _ in range(2):
        ctx = _context(34)
        sk = ctx.make_secret_key()
        dumps.append(ctx.encrypt(sk, [True, False, True], compressed=True).dumps())
    assert dumps[0] == dumps[1]


def _key_material(seed, k):
    """Secret key, compressed and decompressed cloud key, the TLWE key replayed from the RNG."""
    ctx = _context(seed)
    sk = ctx.make_secret_key(tlwe_mask_size=k)
    cck = ctx.make_cloud_key(sk, compressed=True)
    replay = DeterministicRNG(seed)
    replay.uniform_bool((500,))
    tlwe_key = replay.uniform_bool((k, N))
    assert (cck.seed.view(numpy.int32) == replay.uniform_torus32((8,))).all()
    return ctx, sk, cck, cck.decompress(ctx.thread), tlwe_key


@pytest.fixture(scope='module', params=[1, 2], ids=['k1', 'k2'])
def keys(request):
    return _key_material(700 + request.param, request.param)


def test_bootstrap_key_rows_have_the_expected_phase(keys):
    ctx, sk, cck, ck, S = keys
    k = S.shape[0]
    params = ck.bootstrap_key.bk_params
    tr = _np(ck.bootstrap_key.tgsw.samples.a.coeffs, True).reshape(-1, N)
    raw = O.ntt_inverse_i32(O.ff_mul_prepared(tr, numpy.ones_like(tr)))   # undo tgsw_transform_samples
    raw = raw.reshape(500, k + 1, params.decomp_length, k + 1, N)
    assert (raw[..., k, :] == _np(cck.bk_body)).all()
    masks = seeded_uniform(cck.seed, C.NONCE_BOOTSTRAP_KEY, (500, k + 1, params.decomp_length, k, N))
    assert (raw[..., :k, :] == masks).all()
    phase = raw[..., k, :].astype(numpy.int64)
    for u in range(k):
        phase -= O.poly_mul_i32(S[u], numpy.ascontiguousarray(raw[..., u, :])).astype(numpy.int64)
    m = _np(sk.lwe_key.key).astype(numpy.int64)
    h = params.base_powers.astype(numpy.int64)
    want = numpy.zeros_like(phase)
    for mi in range(k):
        want[:, mi] = -m[:, None, None] * h[None, :, None] * S[mi][None, None, :]
    want[:, k, :, 0] = m[:, None] * h[None, :]
    err = _wrap(phase - want).astype(numpy.int64)
    sigma = params.tlwe_params.min_noise * 2**32
    assert numpy.abs(err).max() <= 8 * sigma
    assert err.std() > 0.5 * sigma                                # the rows are noisy, not trivial
    assert (_np(ck.bootstrap_key.tgsw.samples.current_variances) == numpy.float32(params.tlwe_params.min_noise**2)).all()


def test_keyswitch_key_rows_have_the_expected_phase(keys):
    ctx, sk, cck, ck, S = keys
    ks = ck.keyswitch_key.lwe
    a, b, cv = _np(ks.a), _np(ks.b), _np(ks.current_variances)
    in_size, t, base, n = a.shape
    assert in_size == S.size and n == 500
    assert (a[:, :, 0] == 0).all() and (b[:, :, 0] == 0).all() and (cv[:, :, 0] == 0).all()
    assert (a[:, :, 1:] == seeded_uniform(cck.seed, C.NONCE_KEYSWITCH_KEY, (in_size, t, base - 1, n))).all()
    noise = sk.params.in_out_params.min_noise
    assert (cv[:, :, 1:] == numpy.float32(noise**2)).all()
    assert (b == _np(cck.ks_b)).all()
    log2_base = ck.keyswitch_key.log2_base
    phase = b.astype(numpy.int64) - (a.astype(numpy.int64) * _np(sk.lwe_key.key).astype(numpy.int64)).sum(-1)
    hs = numpy.arange(base, dtype=numpy.int64)[None, None, :]
    js = numpy.arange(t, dtype=numpy.int64)[None, :, None]
    want = S.reshape(-1).astype(numpy.int64)[:, None, None] * hs * 2**(32 - (js + 1) * log2_base)
    err = _wrap(phase - want).astype(numpy.int64)[:, :, 1:]
    sigma = noise * 2**32
    assert numpy.abs(err).max() <= 8 * sigma
    assert err.std() > 0.5 * sigma


def test_compressed_cloud_key_serialization_and_sizes(keys):
    ctx, sk, cck, ck, S = keys
    s = cck.dumps()
    back = ctx.load_compressed_cloud_key(s)
    assert back == cck
    assert back.decompress(ctx.thread) == ck
    k = S.shape[0]
    assert len(s) < 500 * (k + 1) * 2 * N * 4 + S.size * 8 * 4 * 4 + 4096
    with pytest.raises(ValueError):
        nufhe_b200.CompressedLweSampleArray.loads(s, ctx.thread)


def test_gate_nand_on_a_decompressed_cloud_key():
    ctx, sk, cck, ck, _ = _key_material(41, 1)
    vm = ctx.make_virtual_machine(ck)
    x = numpy.arange(16) % 2 == 1
    y = numpy.arange(16) // 2 % 2 == 1
    cx = ctx.encrypt(sk, x, compressed=True).decompress(ctx.thread)
    cy = ctx.encrypt(sk, y, compressed=True).decompress(ctx.thread)
    r = vm.gate_nand(cx, cy)
    assert (ctx.decrypt(sk, r) == ~(x & y)).all()
    # the same bits as the oracle's gate with the decompressed key's arrays
    ks = ck.keyswitch_key.device_arrays()
    want = O.gate_binary('nand', (_np(cx.a), _np(cx.b)), (_np(cy.a), _np(cy.b)),
                         _np(ck.bootstrap_key.tgsw.samples.a.coeffs, True), tuple(_np(v) for v in ks))
    assert (_np(r.a) == want[0]).all() and (_np(r.b) == want[1]).all()
