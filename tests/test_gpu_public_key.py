"""Public-key encryption on the GPU: nb_pk_prepare and nb_pk_encrypt against the NumPy restatement (pk_ref.py), bad
arguments, and public-key ciphertexts end to end through gates and lookup tables, sizes and reproducibility."""
import ctypes

import numpy
import pytest
import torch

import pk_ref
from oracle import oracle as O

pytestmark = pytest.mark.gpu
B = 4096
SIGMA = 2**-15 * (2 / numpy.pi)**0.5
VAR = float(numpy.float32(SIGMA**2))


@pytest.fixture(scope='module')
def eng():
    from nufhe_b200.engine import Engine
    return Engine()


def _i32(rng, shape):
    return rng.randint(-2**31, 2**31, size=shape, dtype=numpy.int64).astype(numpy.int32)


def _key(m, n, kind, seed):
    rng = numpy.random.RandomState(seed)
    masks, pk_b = _i32(rng, (m, n)), _i32(rng, m)
    if kind == 'max':
        masks[:] = -1
        pk_b[:] = -2**31
    return masks, pk_b


def _r(m, batch, kind, seed):
    words = _i32(numpy.random.RandomState(seed), (batch, m // 32))
    if kind == 'ones':
        words[:] = -1
    elif kind == 'first_bit':
        words[:] = 0
        words[:, 0] = 1
    elif kind == 'last_bit':
        words[:] = 0
        words[:, -1] = -2**31
    return words


def _run(eng, masks, pk_b, words, mus):
    m, n = masks.shape
    planes = eng.pk_prepare(eng.to_device(masks), eng.to_device(pk_b))
    got = eng.public_encrypt(eng.to_device(words), planes, m, n, eng.to_device(mus), VAR)
    want = pk_ref.encrypt(masks, pk_b, words, mus, VAR)
    for g, w in zip(got, want):
        g = eng.to_host(g)
        assert g.shape == w.shape and (g.view(numpy.uint32) == w.view(numpy.uint32)).all()


@pytest.mark.parametrize('batch', [1, 17, 129, 700, B])
def test_kernel_matches_the_restatement(eng, batch):
    masks, pk_b = _key(16384, 500, 'random', 1)
    _run(eng, masks, pk_b, _r(16384, batch, 'random', batch), _i32(numpy.random.RandomState(batch), batch))


@pytest.mark.parametrize('key_kind, r_kind', [('max', 'ones'), ('max', 'random'), ('random', 'ones'),
                                              ('random', 'first_bit'), ('random', 'last_bit')])
def test_kernel_on_adversarial_keys(eng, key_kind, r_kind):
    masks, pk_b = _key(16384, 500, key_kind, 2)
    _run(eng, masks, pk_b, _r(16384, 129, r_kind, 3), _i32(numpy.random.RandomState(4), 129))


@pytest.mark.parametrize('m', [32, 1056])
@pytest.mark.parametrize('batch', [17, 700])
def test_kernel_other_key_sizes(eng, m, batch):
    masks, pk_b = _key(m, 500, 'random', m)
    _run(eng, masks, pk_b, _r(m, batch, 'random', m + batch), _i32(numpy.random.RandomState(m), batch))
    masks, pk_b = _key(m, 500, 'max', m)
    _run(eng, masks, pk_b, _r(m, batch, 'ones', m), _i32(numpy.random.RandomState(m), batch))


@pytest.mark.parametrize('m, n', [(1056, 500), (64, 7), (16384, 500)])
def test_prepare_matches_a_numpy_relayout(eng, m, n):
    masks, pk_b = _key(m, n, 'random', 5)
    planes = eng.to_host(eng.pk_prepare(eng.to_device(masks), eng.to_device(pk_b)))
    assert planes.size == eng.lib.nb_pk_planes_bytes(m, n)
    assert (planes == pk_ref.planes(masks, pk_b)).all()


def test_bad_arguments_are_rejected(eng):
    from nufhe_b200 import _native
    lib, h = eng.lib, eng.handle
    m, n = 64, 500
    masks, pk_b = _key(m, n, 'random', 6)
    a, b = eng.to_device(masks), eng.to_device(pk_b)
    planes = eng.pk_prepare(a, b)
    words = eng.to_device(_r(m, 4, 'random', 7))
    mus = torch.zeros(4, dtype=torch.int32, device=eng.device)
    out_a = torch.zeros((4, n), dtype=torch.int32, device=eng.device)
    out_b = torch.zeros(4, dtype=torch.int32, device=eng.device)
    out_cv = torch.zeros(4, dtype=torch.float32, device=eng.device)
    p = lambda t: ctypes.c_void_p(t.data_ptr())     # noqa: E731
    v = ctypes.c_float(VAR)
    args = [p(words), p(planes), m, n, p(mus), v, p(out_a), p(out_b), p(out_cv), 4]
    assert lib.nb_pk_encrypt(h, *args) == _native.NB_OK
    for i in (0, 1, 4, 6, 7, 8):                                  # each required pointer NULL
        bad = list(args)
        bad[i] = None
        assert lib.nb_pk_encrypt(h, *bad) == _native.NB_EINVAL
    for bad_m in (0, 48, 33, 1 << 24):                            # not a multiple of 32, or m * 255 >= 2^31
        bad = list(args)
        bad[2] = bad_m
        assert lib.nb_pk_encrypt(h, *bad) == _native.NB_EINVAL
        assert lib.nb_pk_prepare(h, p(a), p(b), bad_m, n, p(planes)) == _native.NB_EINVAL
    bad = list(args)
    bad[3] = 0
    assert lib.nb_pk_encrypt(h, *bad) == _native.NB_EINVAL
    assert lib.nb_pk_prepare(h, None, p(b), m, n, p(planes)) == _native.NB_EINVAL
    assert lib.nb_pk_prepare(h, p(a), p(b), m, n, None) == _native.NB_EINVAL
    bad = list(args)
    bad[-1] = 0
    out_b.fill_(7)
    assert lib.nb_pk_encrypt(h, *bad) == _native.NB_OK            # batch 0: nothing written
    torch.cuda.synchronize()
    assert (out_b == 7).all()
    with pytest.raises(ValueError):
        eng.pk_prepare(a[:33], b[:33])
    with pytest.raises(ValueError):
        eng.public_encrypt(words, planes, 48, n, mus, VAR)
    with pytest.raises(ValueError):
        eng.public_encrypt(words[:3], planes, m, n, mus, VAR)
    ra, rb, rcv = eng.public_encrypt(words[:0], planes, m, n, mus[:0], VAR)
    assert ra.shape == (0, n) and rb.shape == (0,) and rcv.shape == (0,)


# ---------------------------------------------------------------- the Python layer

@pytest.fixture(scope='module')
def api():
    import nufhe_b200
    ctx = nufhe_b200.Context(rng=nufhe_b200.DeterministicRNG(6174))
    sk = ctx.make_secret_key()
    pk = ctx.load_public_key(ctx.make_public_key(sk).dumps())
    ck = ctx.make_cloud_key(sk)
    return nufhe_b200, ctx, sk, pk, ck, ctx.make_virtual_machine(ck)


def test_public_key_ciphertexts_decrypt(api):
    nufhe, ctx, sk, pk, ck, vm = api
    bits = numpy.random.RandomState(8).randint(0, 2, 65536).astype(bool)
    ct = ctx.encrypt(pk, bits)
    assert isinstance(ct, nufhe.LweSampleArray) and tuple(ct.a.shape) == (65536, 500)
    assert (ctx.decrypt(sk, ct) == bits).all()
    cv = ct.current_variances.cpu().numpy()
    assert cv.min() > 0.45 * pk.size * VAR and cv.max() < 0.55 * pk.size * VAR
    with pytest.raises(ValueError):
        ctx.encrypt(pk, bits[:4], compressed=True)


def _pick(rng, count):
    pick = numpy.sort(rng.choice(B, count, replace=False))
    pick[0], pick[-1] = 0, B - 1
    return pick


def test_gates_on_public_key_ciphertexts(api):
    nufhe, ctx, sk, pk, ck, vm = api
    rng = numpy.random.RandomState(9)
    bits = rng.randint(0, 2, (3, B)).astype(bool)
    cts = [ctx.encrypt(pk, v) for v in bits]
    r = vm.gate_nand(cts[0], cts[1])
    assert (ctx.decrypt(sk, r) == ~(bits[0] & bits[1])).all()
    assert (ctx.decrypt(sk, vm.gate_xor(cts[0], cts[1])) == (bits[0] ^ bits[1])).all()
    assert (ctx.decrypt(sk, vm.gate_mux(*cts)) == numpy.where(bits[0], bits[1], bits[2])).all()
    pick = _pick(rng, 48)
    host = [(c.a.cpu().numpy(), c.b.cpu().numpy()) for c in cts[:2]]
    bk = ck.bootstrap_key.tgsw.samples.a.coeffs.cpu().numpy().view(numpy.uint64)
    ks = tuple(v.cpu().numpy() for v in ck.keyswitch_key.device_arrays())
    want = O.gate_binary('nand', (host[0][0][pick], host[0][1][pick]), (host[1][0][pick], host[1][1][pick]), bk, ks)
    assert (r.a.cpu().numpy()[pick] == want[0]).all() and (r.b.cpu().numpy()[pick] == want[1]).all()


def test_luts_on_public_key_ciphertexts(api):
    nufhe, ctx, sk, pk, ck, vm = api
    rng = numpy.random.RandomState(10)
    for bits in (1, 2):
        m = rng.randint(0, 2**bits, B)
        cm = ctx.encrypt_int(pk, m, bits)
        assert (ctx.decrypt_int(sk, cm, bits) == m).all()
        f = (numpy.arange(2**bits) * 3 + 1) % 2**bits
        assert (ctx.decrypt_int(sk, vm.lut(vm.make_lut(f, bits), cm), bits) == f[m]).all()
    a, b = rng.randint(0, 2, B), rng.randint(0, 2, B)
    xa, xb = ctx.encrypt_int(pk, a, 2), ctx.encrypt_int(pk, b, 2)
    s, c = vm.lut(vm.make_lut([[0, 1, 0, 1], [0, 0, 1, 1]], 2), vm.int_add(xa, xb))
    assert (ctx.decrypt_int(sk, s, 2) == (a + b) % 2).all() and (ctx.decrypt_int(sk, c, 2) == (a + b) // 2).all()


def test_mask_size_2_key():
    import nufhe_b200
    ctx = nufhe_b200.Context(rng=nufhe_b200.DeterministicRNG(79))
    sk = ctx.make_secret_key(tlwe_mask_size=2)
    pk = ctx.make_public_key(sk)
    vm = ctx.make_virtual_machine(ctx.make_cloud_key(sk))
    x, y = numpy.arange(16) % 2 == 1, numpy.arange(16) // 2 % 2 == 1
    cx, cy = ctx.encrypt(pk, x), ctx.encrypt(pk, y)
    assert (ctx.decrypt(sk, vm.gate_nand(cx, cy)) == ~(x & y)).all()
    assert (ctx.decrypt(sk, vm.gate_or(cx, cy)) == (x | y)).all()


def test_seeded_contexts_give_identical_dumps():
    import nufhe_b200
    dumps = []
    for _ in range(2):
        ctx = nufhe_b200.Context(rng=nufhe_b200.DeterministicRNG(98))
        sk = ctx.make_secret_key()
        pk = ctx.make_public_key(sk)
        dumps.append((pk.dumps(), ctx.encrypt(pk, numpy.arange(100) % 3 == 0).dumps()))
    assert dumps[0] == dumps[1]
    assert len(dumps[0][0]) <= 70e3, len(dumps[0][0])
