"""Result packing on the GPU: nb_pack_digits, nb_ntt_mac and nb_pack_finish bit-exact against the NumPy restatement
(pack_ref.py) or Python integers, including inputs at the 2^58 exactness bound, bad arguments, the whole vm.pack against
the restatement, packed gate / LUT / public-key / k = 2 results end to end through pickles, the size of 4096 packed
bits, and the noise packing adds (DESIGN.md section 12)."""
import ctypes

import numpy
import pytest
import torch

import pack_ref

pytestmark = pytest.mark.gpu
P = 0xffffffff00000001
N = 1024


@pytest.fixture(scope='module')
def eng():
    from nufhe_b200.engine import Engine
    return Engine()


@pytest.fixture(scope='module')
def api():
    import nufhe_b200
    ctx = nufhe_b200.Context(rng=nufhe_b200.DeterministicRNG(121))
    sk = ctx.make_secret_key()
    ck = ctx.make_cloud_key(sk)
    vm = ctx.make_virtual_machine(ck)
    psk, pk = ctx.make_packing_keys(sk)
    return nufhe_b200, ctx, sk, vm, psk, pk


def _i32(rng, shape):
    return rng.randint(-2**31, 2**31, size=shape, dtype=numpy.int64).astype(numpy.int32)


def _u64(rng, shape):
    return (rng.randint(0, 2**32, size=shape, dtype=numpy.uint64) << numpy.uint64(32)
            | rng.randint(0, 2**32, size=shape, dtype=numpy.uint64)) % numpy.uint64(P)


@pytest.mark.parametrize('batch', [1, 31, 1024, 1025, 5000])
def test_pack_digits_kernel(eng, batch):
    rng = numpy.random.RandomState(batch)
    a = _i32(rng, (batch, 500))
    a[0, :7] = pack_ref.i32([0, 2**15 - 1, 2**15, 0x7fff8000, 0xffff8000, -1, 2**31])
    got = eng.to_host(eng.pack_digits(eng.to_device(a)))
    G = -(-batch // N)
    want = numpy.zeros((G * N, 500, 2), numpy.int64)
    want[:batch] = pack_ref.digits(a)
    want = want.reshape(G, N, 1000).transpose(0, 2, 1)
    assert got.shape == (G, 1000, N) and (got == want).all()


@pytest.mark.parametrize('G, R, U', [(1, 1, 1), (2, 37, 3), (3, 1000, 2), (1, 2, 1)])
def test_ntt_mac_kernel_matches_python_integers(eng, G, R, U):
    rng = numpy.random.RandomState(G * 1000 + R)
    x, key = _u64(rng, (G, R, N)), _u64(rng, (R, U, N))
    x[0, 0, :4] = P - 1
    key[0, 0, :4] = P - 1
    got = eng.to_host(eng.ntt_mac(eng.to_device(x), eng.to_device(key)), unsigned=True)
    cols = [0, 1, 2, 3, 511, 1022, 1023] if R > 40 else range(N)
    xo, ko = x.astype(object), key.astype(object)
    for g in range(G):
        for u in range(U):
            for c in cols:
                assert int(got[g, u, c]) == int(sum(xo[g, :, c] * ko[:, u, c]) % P)


def test_transform_chain_at_the_exactness_bound(eng):
    """Every digit -128 and every key coefficient -2^31: each coefficient of C is 1000 * 2^38 * (2 (y + 1) - N), up to
    1000 * 2^48 < 2^58 at y = N - 1; forward NTT, MAC and centred inverse give it exactly mod 2^32."""
    R, U = 1000, 2
    digits = torch.full((1, R, N), -128, dtype=torch.int32, device=eng.device)
    keys = torch.full((R, U, N), -2**31, dtype=torch.int32, device=eng.device)
    c = eng.to_host(eng.ntt_inverse_i32(eng.ntt_mac(eng.ntt_forward_i32(digits), eng.ntt_forward_i32(keys))))
    y = numpy.arange(N)
    want = pack_ref.i32([R * 128 * 2**31 * (2 * (int(v) + 1) - N) for v in y])
    assert (c[0] == want[None, :]).all()


@pytest.mark.parametrize('batch, k', [(1, 1), (1025, 1), (5000, 1), (1500, 2)])
def test_pack_finish_kernel(eng, batch, k):
    rng = numpy.random.RandomState(batch + k)
    G = -(-batch // N)
    c, b = _i32(rng, (G, k + 1, N)), _i32(rng, batch)
    c[0, 0, :4] = pack_ref.i32([0, 2**15, -2**15, 2**31])
    got = eng.to_host(eng.pack_finish(eng.to_device(c), eng.to_device(b)))
    assert got.dtype == numpy.uint16 and (got == pack_ref.finish(c.astype(numpy.int64), b)).all()


def test_bad_arguments_are_rejected(eng):
    lib, h = eng.lib, eng.handle
    from nufhe_b200 import _native
    a = eng.to_device(numpy.zeros((4, 500), numpy.int32))
    d = torch.empty((1, 1000, N), dtype=torch.int32, device=eng.device)
    x = torch.zeros((1, 2, N), dtype=torch.int64, device=eng.device)
    key = torch.zeros((2, 1, N), dtype=torch.int64, device=eng.device)
    out = torch.empty((1, 1, N), dtype=torch.int64, device=eng.device)
    c = torch.zeros((1, 2, N), dtype=torch.int32, device=eng.device)
    b = torch.zeros(4, dtype=torch.int32, device=eng.device)
    o16 = torch.empty((1, 2, N), dtype=torch.uint16, device=eng.device)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    bad = [('nb_pack_digits', (None, 500, p(d), 4)), ('nb_pack_digits', (p(a), 500, None, 4)),
           ('nb_pack_digits', (p(a), 0, p(d), 4)), ('nb_pack_digits', (p(a), 500, p(d), 2048 * N + 1)),
           ('nb_ntt_mac', (None, p(key), p(out), 2, 1, 1)), ('nb_ntt_mac', (p(x), None, p(out), 2, 1, 1)),
           ('nb_ntt_mac', (p(x), p(key), None, 2, 1, 1)), ('nb_ntt_mac', (p(x), p(key), p(out), 0, 1, 1)),
           ('nb_ntt_mac', (p(x), p(key), p(out), 2, 0, 1)),
           ('nb_pack_finish', (None, p(b), 1, p(o16), 4)), ('nb_pack_finish', (p(c), None, 1, p(o16), 4)),
           ('nb_pack_finish', (p(c), p(b), 1, None, 4)), ('nb_pack_finish', (p(c), p(b), 0, p(o16), 4))]
    for name, args in bad:
        assert getattr(lib, name)(h, *args) == _native.NB_EINVAL, (name, args)
    # an empty batch is a no-op
    assert lib.nb_pack_digits(h, p(a), 500, p(d), 0) == _native.NB_OK
    assert lib.nb_ntt_mac(h, p(x), p(key), p(out), 2, 1, 0) == _native.NB_OK
    assert lib.nb_pack_finish(h, p(c), p(b), 1, p(o16), 0) == _native.NB_OK
    eng.synchronize()
    with pytest.raises(ValueError):
        eng.ntt_mac(x, torch.zeros((3, 1, N), dtype=torch.int64, device=eng.device))


def _key_polys(pk):
    from chacha_ref import seeded_uniform
    k = pk.params.tgsw_params.tlwe_params.mask_size
    return pack_ref.key_polys(seeded_uniform(pk.seed, 4, (500, 2, k, N)), pk.body.cpu().numpy())


@pytest.mark.parametrize('batch', [1, 1024, 1025, 4096, 5000])
def test_vm_pack_matches_the_restatement(api, batch):
    nufhe, ctx, sk, vm, psk, pk = api
    rng = numpy.random.RandomState(batch)
    a, b = _i32(rng, (batch, 500)), _i32(rng, batch)
    ct = nufhe.LweSampleArray(sk.params.in_out_params, ctx.thread.to_device(a), ctx.thread.to_device(b),
                              torch.zeros(batch, dtype=torch.float32, device=ctx.thread.device))
    packed = vm.pack(pk, ct)
    assert (packed.data.cpu().numpy() == pack_ref.pack(a, b, _key_polys(pk))).all()
    ph = nufhe.packing.packed_phases(ctx.thread, psk, packed)
    assert (ph == pack_ref.phases(packed.data.cpu().numpy(), psk.key.cpu().numpy())[:batch]).all()


def _round_trip(ctx, packed):
    return ctx.load_packed_ciphertext(packed.dumps())


def test_gate_outputs_end_to_end(api):
    nufhe, ctx, sk, vm, psk, pk = api
    rng = numpy.random.RandomState(3)
    x, y = rng.randint(0, 2, (2, 4096)).astype(bool)
    r = vm.gate_nand(ctx.encrypt(sk, x), ctx.encrypt(sk, y))
    packed = vm.pack(ctx.load_packing_key(pk.dumps()), r)
    s = packed.dumps()
    assert len(s) <= 16384 + 1024
    back = ctx.load_packed_ciphertext(s)
    psk2 = ctx.load_packing_secret_key(psk.dumps())
    assert (ctx.decrypt(psk2, back) == ~(x & y)).all()
    assert (ctx.decrypt(sk, r) == ~(x & y)).all()
    with pytest.raises(TypeError):
        ctx.decrypt(sk, back)
    with pytest.raises(TypeError):
        ctx.decrypt(psk, r)


def test_lut_outputs_end_to_end(api):
    nufhe, ctx, sk, vm, psk, pk = api
    rng = numpy.random.RandomState(4)
    a, b = rng.randint(0, 2, (2, 4096))
    s, c = vm.lut(vm.make_lut([[0, 1, 0, 1], [0, 0, 1, 1]], 2), vm.int_add(ctx.encrypt_int(sk, a, 2),
                                                                          ctx.encrypt_int(sk, b, 2)))
    back = _round_trip(ctx, vm.pack(pk, nufhe.concatenate([s, c])))      # sums, then carries
    got = ctx.decrypt_int(psk, back, 2)
    assert got.shape == (8192,) and (got[:4096] == (a + b) % 2).all() and (got[4096:] == (a + b) // 2).all()


def test_public_key_inputs_on_a_decompressed_cloud_key(api):
    nufhe, ctx, sk, vm, psk, pk = api
    pub = ctx.make_public_key(sk)
    vm2 = ctx.make_virtual_machine(ctx.make_cloud_key(sk, compressed=True).decompress(ctx.thread))
    rng = numpy.random.RandomState(5)
    x, y = rng.randint(0, 2, (2, 4096)).astype(bool)
    r = vm2.gate_or(ctx.encrypt(pub, x), ctx.encrypt(pub, y))
    assert (ctx.decrypt(psk, _round_trip(ctx, vm2.pack(pk, r))) == (x | y)).all()


def test_mask_size_2_key():
    import nufhe_b200
    ctx = nufhe_b200.Context(rng=nufhe_b200.DeterministicRNG(122))
    sk = ctx.make_secret_key(tlwe_mask_size=2)
    vm = ctx.make_virtual_machine(ctx.make_cloud_key(sk))
    psk, pk = ctx.make_packing_keys(sk)
    rng = numpy.random.RandomState(6)
    x, y = rng.randint(0, 2, (2, 1100)).astype(bool)
    r = vm.gate_nand(ctx.encrypt(sk, x), ctx.encrypt(sk, y))
    packed = vm.pack(pk, r)
    assert tuple(packed.data.shape) == (2, 3, N)
    assert (packed.data.cpu().numpy() == pack_ref.pack(r.a.cpu().numpy(), r.b.cpu().numpy(), _key_polys(pk))).all()
    assert (ctx.decrypt(psk, _round_trip(ctx, packed)) == ~(x & y)).all()
    with pytest.raises(ValueError):
        ctx.make_virtual_machine(ctx.make_cloud_key(sk)).pack(
            ctx.make_packing_keys(ctx.make_secret_key())[1], r)


def test_packing_noise(api):
    """Packed phase minus LWE phase over 65 536 gate outputs: sample variance within 0.5 - 2 times the DESIGN.md
    estimate (pack_ref.noise_terms), nothing beyond 7 sigma."""
    nufhe, ctx, sk, vm, psk, pk = api
    rng = numpy.random.RandomState(7)
    x, y = rng.randint(0, 2, (2, 65536)).astype(bool)
    r = vm.gate_nand(ctx.encrypt(sk, x), ctx.encrypt(sk, y))
    packed = vm.pack(pk, r)
    from nufhe_b200.packing import packed_phases
    from nufhe_b200.lwe import lwe_decrypt
    diff = pack_ref.i32(packed_phases(ctx.thread, psk, packed).astype(numpy.int64)
                        - lwe_decrypt(ctx.thread, r, sk.lwe_key).astype(numpy.int64)).astype(numpy.float64) * 2.0**-32
    est = sum(pack_ref.noise_terms(sk.params))
    var = float(diff.var())
    print('packing noise: measured variance %.4g, estimate %.4g (ratio %.3f), max |err| %.2f sigma'
          % (var, est, var / est, numpy.abs(diff).max() / est**0.5))
    assert 0.5 * est <= var <= 2 * est
    assert numpy.abs(diff).max() <= 7 * est**0.5
    assert (ctx.decrypt(psk, packed) == ~(x & y)).all()
