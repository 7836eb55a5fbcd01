"""Compressed keys and ciphertexts on the GPU: nb_seeded_uniform_i32 against the NumPy keystream (chacha_ref.py), and
compressed ciphertexts and cloud keys end to end -- decompression, gates and lookup tables on them, sizes and
reproducibility."""
import ctypes

import numpy
import pytest
import torch

from chacha_ref import chacha20_words
from oracle import oracle as O

pytestmark = pytest.mark.gpu
N = 1024
B = 4096


@pytest.fixture(scope='module')
def eng():
    from nufhe_b200.engine import Engine
    return Engine()


def _seed(rng):
    return rng.randint(0, 2**32, size=8, dtype=numpy.uint64).astype(numpy.uint32)


@pytest.mark.parametrize('nonce, first, count', [
    (0, 0, 1), (0, 0, 15), (0, 0, 17), (5, 0, 1000003),               # counts that are not multiples of 16
    (0, 5, 11), (3, 16 * 7 + 9, 500), (2**64 - 1, 123457, 77777),       # first mid-block, nonce != 0
    (1, 16 * (2**32 - 1) + 3, 100),                                     # the carry from counter word 12 into word 13
    (2, 16 * 2**32 - 37, 100003),
    (7, 2**64 - 16 * 3 - 5, 16 * 3 + 5),                                # the last words of the stream
])
def test_kernel_matches_the_reference(eng, nonce, first, count):
    seed = _seed(numpy.random.RandomState(count % 997))
    got = eng.to_host(eng.seeded_uniform(seed, nonce, (count,), first=first))
    assert (got == chacha20_words(seed, nonce, first, count)).all()


def test_kernel_full_keyswitch_key_mask(eng):
    """The key-switch key's mask (1024, 8, 3, 500), and all of ks_a's size (1024, 8, 4, 500): 16.4 M words."""
    seed = _seed(numpy.random.RandomState(2))
    for shape in ((1024, 8, 3, 500), (1024, 8, 4, 500)):
        got = eng.to_host(eng.seeded_uniform(seed, 2, shape))
        assert got.shape == shape
        assert (got.reshape(-1) == chacha20_words(seed, 2, 0, int(numpy.prod(shape)))).all()


def test_bad_arguments_are_rejected(eng):
    from nufhe_b200 import _native
    seed = numpy.arange(8, dtype=numpy.uint32)
    out = torch.zeros(64, dtype=torch.int32, device=eng.device)
    lib, sp = eng.lib, seed.ctypes.data_as(ctypes.c_void_p)
    ptr = ctypes.c_void_p(out.data_ptr())
    assert lib.nb_seeded_uniform_i32(eng.handle, None, 0, 0, ptr, 16) == _native.NB_EINVAL
    assert lib.nb_seeded_uniform_i32(eng.handle, sp, 0, 0, None, 16) == _native.NB_EINVAL
    assert lib.nb_seeded_uniform_i32(eng.handle, sp, 0, 2**64 - 10, ptr, 11) == _native.NB_EINVAL
    assert lib.nb_seeded_uniform_i32(eng.handle, sp, 0, 2**63, ptr, 2**63 + 1) == _native.NB_EINVAL
    assert lib.nb_seeded_uniform_i32(eng.handle, sp, 0, 2**64 - 10, ptr, 10) == _native.NB_OK
    assert (eng.to_host(out[:10]) == chacha20_words(seed, 0, 2**64 - 10, 10)).all()
    with pytest.raises(ValueError):
        eng.seeded_uniform(seed, 0, (11,), first=2**64 - 10)
    with pytest.raises(ValueError):
        eng.seeded_uniform(seed[:7], 0, (11,))
    assert eng.seeded_uniform(seed, 0, (0, 500)).shape == (0, 500)


# ---------------------------------------------------------------- the Python layer

@pytest.fixture(scope='module')
def api():
    import nufhe_b200
    ctx = nufhe_b200.Context(rng=nufhe_b200.DeterministicRNG(5150))
    sk = ctx.make_secret_key()
    cck = ctx.make_cloud_key(sk, compressed=True)
    ck = cck.decompress(ctx.thread)
    return nufhe_b200, ctx, sk, cck, ck, ctx.make_virtual_machine(ck)


def test_compressed_ciphertexts_through_gates_and_luts(api):
    nufhe, ctx, sk, cck, ck, vm = api
    rng = numpy.random.RandomState(3)
    x, y = rng.randint(0, 2, B).astype(bool), rng.randint(0, 2, B).astype(bool)
    cx, cy = ctx.encrypt(sk, x, compressed=True), ctx.encrypt(sk, y, compressed=True)
    assert isinstance(cx, nufhe.CompressedLweSampleArray)
    dx, dy = ctx.load_compressed_ciphertext(cx.dumps()).decompress(ctx.thread), cy.decompress(ctx.thread)
    assert (ctx.decrypt(sk, dx) == x).all() and (ctx.decrypt(sk, dy) == y).all()
    assert (ctx.decrypt(sk, vm.gate_nand(dx, dy)) == ~(x & y)).all()
    assert (ctx.decrypt(sk, vm.gate_xor(dx, dy)) == (x ^ y)).all()
    for bits in (1, 2):
        m = rng.randint(0, 2**bits, B)
        cm = ctx.encrypt_int(sk, m, bits, compressed=True)
        dm = ctx.load_compressed_ciphertext(cm.dumps()).decompress(ctx.thread)
        assert (ctx.decrypt_int(sk, dm, bits) == m).all()
        f = (numpy.arange(2**bits) * 3 + 1) % 2**bits
        assert (ctx.decrypt_int(sk, vm.lut(vm.make_lut(f, bits), dm), bits) == f[m]).all()


def _pick(rng, count):
    pick = numpy.sort(rng.choice(B, count, replace=False))
    pick[0], pick[-1] = 0, B - 1
    return pick


def test_gates_on_a_decompressed_key_match_the_oracle(api):
    """B = 4096 on the GPU; the oracle recomputes 48 NAND and 24 MUX outputs spread over the batch with the decompressed
    key's own arrays (about 0.1 s per bootstrap on the CPU)."""
    nufhe, ctx, sk, cck, ck, vm = api
    rng = numpy.random.RandomState(4)
    bits = rng.randint(0, 2, (3, B)).astype(bool)
    cts = [ctx.encrypt(sk, v, compressed=True).decompress(ctx.thread) for v in bits]
    host = [(cts[i].a.cpu().numpy(), cts[i].b.cpu().numpy()) for i in range(3)]
    bk = ck.bootstrap_key.tgsw.samples.a.coeffs.cpu().numpy().view(numpy.uint64)
    ks = tuple(v.cpu().numpy() for v in ck.keyswitch_key.device_arrays())

    r = vm.gate_nand(cts[0], cts[1])
    assert (ctx.decrypt(sk, r) == ~(bits[0] & bits[1])).all()
    pick = _pick(rng, 48)
    want = O.gate_binary('nand', (host[0][0][pick], host[0][1][pick]), (host[1][0][pick], host[1][1][pick]), bk, ks)
    assert (r.a.cpu().numpy()[pick] == want[0]).all() and (r.b.cpu().numpy()[pick] == want[1]).all()

    r = vm.gate_mux(cts[0], cts[1], cts[2])
    assert (ctx.decrypt(sk, r) == numpy.where(bits[0], bits[1], bits[2])).all()
    pick = _pick(rng, 24)
    want = O.gate_mux(*[(h[0][pick], h[1][pick]) for h in host], bk, ks)
    assert (r.a.cpu().numpy()[pick] == want[0]).all() and (r.b.cpu().numpy()[pick] == want[1]).all()


def test_two_output_lut_on_a_decompressed_key(api):
    nufhe, ctx, sk, cck, ck, vm = api
    rng = numpy.random.RandomState(5)
    a, b = rng.randint(0, 2, B), rng.randint(0, 2, B)
    xa, xb = ctx.encrypt_int(sk, a, 2), ctx.encrypt_int(sk, b, 2)
    s, c = vm.lut(vm.make_lut([[0, 1, 0, 1], [0, 0, 1, 1]], 2), vm.int_add(xa, xb))
    assert (ctx.decrypt_int(sk, s, 2) == (a + b) % 2).all() and (ctx.decrypt_int(sk, c, 2) == (a + b) // 2).all()


def test_mask_size_2_compressed_key():
    import nufhe_b200
    ctx = nufhe_b200.Context(rng=nufhe_b200.DeterministicRNG(78))
    sk = ctx.make_secret_key(tlwe_mask_size=2)
    ck = ctx.load_compressed_cloud_key(ctx.make_cloud_key(sk, compressed=True).dumps()).decompress(ctx.thread)
    vm = ctx.make_virtual_machine(ck)
    x, y = numpy.arange(16) % 2 == 1, numpy.arange(16) // 2 % 2 == 1
    cx, cy = (ctx.encrypt(sk, v, compressed=True).decompress(ctx.thread) for v in (x, y))
    assert (ctx.decrypt(sk, vm.gate_nand(cx, cy)) == ~(x & y)).all()
    assert (ctx.decrypt(sk, vm.gate_or(cx, cy)) == (x | y)).all()


def test_sizes(api):
    nufhe, ctx, sk, cck, ck, vm = api
    compressed_key, full_key = len(cck.dumps()), len(ck.dumps())
    assert compressed_key <= 8.4e6 and full_key > 98e6, (compressed_key, full_key)
    bits = numpy.ones(B, bool)
    compressed_ct, full_ct = len(ctx.encrypt(sk, bits, compressed=True).dumps()), len(ctx.encrypt(sk, bits).dumps())
    assert compressed_ct <= 20e3 and full_ct > 8e6, (compressed_ct, full_ct)


def test_seeded_contexts_give_identical_dumps():
    import nufhe_b200
    dumps = []
    for _ in range(2):
        ctx = nufhe_b200.Context(rng=nufhe_b200.DeterministicRNG(99))
        sk = ctx.make_secret_key()
        ck = ctx.make_cloud_key(sk, compressed=True)
        dumps.append((ck.dumps(), ctx.encrypt(sk, numpy.arange(100) % 3 == 0, compressed=True).dumps(),
                      ck.decompress(ctx.thread).dumps()))
    assert dumps[0] == dumps[1]
