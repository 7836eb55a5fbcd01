"""Compact public-key encryption on the GPU: nb_compact_finish and nb_compact_extract bit-exact against the NumPy
restatement (compact_ref.py) with outputs between sentinel guard rows, bad arguments, vm.expand against explicit
extraction and Engine.keyswitch, encrypted bits and integers through gates, LUTs, packing, pickles and other cloud-key
kinds, the pickled sizes, and the noise of expanded samples (DESIGN.md section 16)."""
import ctypes

import numpy
import pytest
import torch

import compact_ref

pytestmark = pytest.mark.gpu
N = 1024
SENTINEL = 0x5a5a5a5a
BOUNDARY = [0, 2**15 - 1, 2**15, 0x7fff8000, 0xffff8000, -1, -2**31]


@pytest.fixture(scope='module')
def eng():
    from nufhe_b200.engine import Engine
    return Engine()


@pytest.fixture(scope='module')
def api():
    import nufhe_b200
    ctx = nufhe_b200.Context(rng=nufhe_b200.DeterministicRNG(131))
    sk = ctx.make_secret_key()
    ck, cpk = ctx.make_cloud_key(sk, compact_public_key=True)
    vm = ctx.make_virtual_machine(ck)
    return nufhe_b200, ctx, sk, ck, cpk, vm


def _p(t, offset=0):
    return ctypes.c_void_p(t.data_ptr() + offset * t.element_size())


def _guarded(eng, count, dtype, guard):
    """A flat buffer of `count` elements between `guard` sentinel elements on each side, and the offset of the body."""
    t = torch.full((count + 2 * guard,), SENTINEL if dtype == torch.int32 else 0x5a5a, dtype=torch.int32, device=eng.device)
    if dtype == torch.uint16:
        t = t.to(torch.int16).view(torch.uint16)
    return t, guard


def _check_guards(t, guard, count, dtype):
    h = t.view(torch.int16).cpu().numpy().view(numpy.uint16) if dtype == torch.uint16 else t.cpu().numpy()
    s = 0x5a5a if dtype == torch.uint16 else SENTINEL
    assert (h[:guard] == s).all() and (h[guard + count:] == s).all()
    return h[guard:guard + count]


@pytest.mark.parametrize('batch, k', [(1, 1), (1000, 1), (3 * N - 5, 1), (64 * N - 300, 1), (3 * N - 5, 2)])
def test_compact_finish_kernel(eng, batch, k):
    rng = numpy.random.RandomState(batch + k)
    G = -(-batch // N)
    c = rng.randint(-2**31, 2**31, size=(G, k + 1, N), dtype=numpy.int64).astype(numpy.int32)
    e1 = rng.randint(-2**20, 2**20, size=(G, k, N)).astype(numpy.int32)
    e2 = rng.randint(-2**20, 2**20, size=(G, N)).astype(numpy.int32)
    mus = rng.randint(-2**31, 2**31, size=batch, dtype=numpy.int64).astype(numpy.int32)
    c[0, :, :7] = compact_ref.i32(BOUNDARY)
    e1[0, :, :7] = 0
    e2[0, :7] = 0
    mus[:min(batch, 7)] = 0
    total = G * (k + 1) * N
    out, off = _guarded(eng, total, torch.uint16, N)
    dev = [eng.to_device(x) for x in (c, e1, e2, mus)]
    assert eng.lib.nb_compact_finish(eng.handle, *[_p(x) for x in dev], k, _p(out, off), batch) == 0
    got = _check_guards(out, off, total, torch.uint16).reshape(G, k + 1, N)
    want = compact_ref.finish(compact_ref.u32(c), e1, e2, mus)
    assert (got == want).all()
    assert list(got[0, 0, :7]) == [0, 0, 1, 0x8000, 0, 0, 0x8000]
    if batch % N:
        assert (got[-1, k, batch % N:] == 0).all()                  # empty body slots
    assert (eng.to_host(eng.compact_finish(*dev)) == want).all()


@pytest.mark.parametrize('rows, k', [(1, 1), (1000, 1), (3 * N - 5, 1), (64 * N - 300, 1), (3 * N - 5, 2)])
def test_compact_extract_kernel(eng, rows, k):
    rng = numpy.random.RandomState(rows + 10 * k)
    G = -(-rows // N)
    data = rng.randint(0, 2**16, size=(G, k + 1, N)).astype(numpy.uint16)
    data[:, :, :4] = [0, 0x7fff, 0x8000, 0xffff]
    data[:, :, -2:] = [0x8000, 0xffff]
    out_a, off_a = _guarded(eng, rows * k * N, torch.int32, k * N)
    out_b, off_b = _guarded(eng, rows, torch.int32, 32)
    d = eng.to_device(data.view(numpy.int16)).view(torch.uint16)
    assert eng.lib.nb_compact_extract(eng.handle, _p(d), k, _p(out_a, off_a), _p(out_b, off_b), rows) == 0
    a = _check_guards(out_a, off_a, rows * k * N, torch.int32).reshape(rows, k * N)
    b = _check_guards(out_b, off_b, rows, torch.int32)
    # every row against the restatement up to 4096 rows, beyond that the boundary slots of every group and a sample
    if rows <= 4096:
        sel = numpy.arange(rows)
        want_a, want_b = compact_ref.extract(data, rows)
    else:
        sel = numpy.unique(numpy.concatenate([(numpy.arange(G)[:, None] * N + numpy.array([0, 1, 31, 32, N - 1])).ravel(),
                                              rng.randint(0, rows, 512), [rows - 1]]))
        sel = sel[sel < rows]
        want_a, want_b = _extract_rows(data, sel)
    assert (a[sel] == want_a).all() and (b[sel] == want_b).all()
    ea, eb = eng.compact_extract(d, rows)
    assert (eng.to_host(ea) == a).all() and (eng.to_host(eb) == b).all()


def _extract_rows(data, rows):
    x = compact_ref.unround16(data).astype(numpy.int64)
    k = data.shape[1] - 1
    j = numpy.arange(N)
    a = numpy.empty((len(rows), k * N), numpy.int64)
    for i, c in enumerate(rows):
        g, p = divmod(int(c), N)
        for u in range(k):
            a[i, u * N:(u + 1) * N] = numpy.where(j <= p, x[g, u, (p - j) % N], -x[g, u, (N + p - j) % N])
    return compact_ref.i32(a), compact_ref.i32(x[rows // N, k, rows % N])


def test_bad_arguments_are_rejected(eng):
    from nufhe_b200 import _native
    lib, h = eng.lib, eng.handle
    c = torch.zeros((1, 2, N), dtype=torch.int32, device=eng.device)
    e1 = torch.zeros((1, 1, N), dtype=torch.int32, device=eng.device)
    e2 = torch.zeros((1, N), dtype=torch.int32, device=eng.device)
    mus = torch.zeros(4, dtype=torch.int32, device=eng.device)
    o16 = torch.zeros((1, 2, N), dtype=torch.int16, device=eng.device)
    oa = torch.empty((4 * N + 4,), dtype=torch.int32, device=eng.device)
    ob = torch.empty((4,), dtype=torch.int32, device=eng.device)
    bad = [('nb_compact_finish', (None, _p(e1), _p(e2), _p(mus), 1, _p(o16), 4)),
           ('nb_compact_finish', (_p(c), None, _p(e2), _p(mus), 1, _p(o16), 4)),
           ('nb_compact_finish', (_p(c), _p(e1), None, _p(mus), 1, _p(o16), 4)),
           ('nb_compact_finish', (_p(c), _p(e1), _p(e2), None, 1, _p(o16), 4)),
           ('nb_compact_finish', (_p(c), _p(e1), _p(e2), _p(mus), 1, None, 4)),
           ('nb_compact_finish', (_p(c), _p(e1), _p(e2), _p(mus), 0, _p(o16), 4)),
           ('nb_compact_extract', (None, 1, _p(oa), _p(ob), 4)),
           ('nb_compact_extract', (_p(o16), 1, None, _p(ob), 4)),
           ('nb_compact_extract', (_p(o16), 1, _p(oa), None, 4)),
           ('nb_compact_extract', (_p(o16), 0, _p(oa), _p(ob), 4)),
           ('nb_compact_extract', (_p(o16, 1), 1, _p(oa), _p(ob), 4)),          # data not 8-byte aligned
           ('nb_compact_extract', (_p(o16), 1, _p(oa, 1), _p(ob), 4)),          # out_a not 16-byte aligned
           ('nb_compact_extract', (_p(o16), 1, _p(oa), _p(ob), 65536 * N + 1))]
    for name, args in bad:
        assert getattr(lib, name)(h, *args) == _native.NB_EINVAL, (name, args)
    assert lib.nb_compact_finish(h, _p(c), _p(e1), _p(e2), _p(mus), 1, _p(o16), 0) == _native.NB_OK
    assert lib.nb_compact_extract(h, _p(o16), 1, _p(oa), _p(ob), 0) == _native.NB_OK
    eng.synchronize()
    with pytest.raises(ValueError):
        eng.compact_finish(c, e1, e2, torch.zeros(2000, dtype=torch.int32, device=eng.device))
    with pytest.raises(ValueError):
        eng.compact_extract(o16.view(torch.uint16), 2000)


@pytest.mark.parametrize('batch, one_group_passes', [(4096, False), (4096, True), (20000, False)])
def test_vm_expand_is_extraction_then_keyswitch(api, monkeypatch, batch, one_group_passes):
    nufhe, ctx, sk, ck, cpk, vm = api
    thr = ctx.thread
    if one_group_passes:
        monkeypatch.setattr(nufhe.compact, 'PASS_BYTES', 4 * N * N)
    bits = numpy.random.RandomState(batch).randint(0, 2, size=batch).astype(bool)
    ct = ctx.encrypt(cpk, bits)
    out = vm.expand(ct)
    a, b = compact_ref.extract(ct.data.cpu().numpy(), batch)
    ra, rb, _ = thr.keyswitch(ck.keyswitch_key.device_arrays(), (thr.to_device(a), thr.to_device(b)))
    assert (out.a.cpu().numpy() == ra.cpu().numpy()).all() and (out.b.cpu().numpy() == rb.cpu().numpy()).all()
    assert (ctx.decrypt(sk, out) == bits).all()


def test_bits_integers_gates_and_luts(api):
    nufhe, ctx, sk, ck, cpk, vm = api
    rng = numpy.random.RandomState(3)
    x, y = rng.randint(0, 2, (2, 4096)).astype(bool)
    cx, cy = vm.expand(ctx.encrypt(cpk, x)), vm.expand(ctx.encrypt(cpk, y))
    assert (ctx.decrypt(sk, cx) == x).all() and (ctx.decrypt(sk, cy) == y).all()
    assert (ctx.decrypt(sk, vm.gate_nand(cx, cy)) == ~(x & y)).all()
    v = rng.randint(0, 4, 4096)
    cv = vm.expand(ctx.encrypt_int(cpk, v, 2))
    assert (ctx.decrypt_int(sk, cv, 2) == v).all()
    table = [3, 0, 2, 1]
    assert (ctx.decrypt_int(sk, vm.lut(vm.make_lut(table, 2), cv), 2) == numpy.array(table)[v]).all()


def test_pickles_sizes_and_packing(api):
    nufhe, ctx, sk, ck, cpk, vm = api
    s = cpk.dumps()
    assert len(s) == 5208                                           # 4 KB body, seed, params
    bits = numpy.random.RandomState(4).randint(0, 2, 4096).astype(bool)
    assert len(ctx.encrypt(cpk, bits).dumps()) == 17199             # 16 KB of data: 4.2 bytes per bit
    c = ctx.encrypt(ctx.load_compact_public_key(s), bits).dumps()
    out = vm.expand(ctx.load_compact_ciphertext(c))
    psk, pk = ctx.make_packing_keys(sk)
    packed = vm.pack(pk, vm.gate_not(out))
    assert (ctx.decrypt(psk, ctx.load_packed_ciphertext(packed.dumps())) == ~bits).all()


@pytest.mark.parametrize('kind', ['compressed', 'multi_bit', 'k2'])
def test_other_cloud_keys(kind):
    import nufhe_b200
    ctx = nufhe_b200.Context(rng=nufhe_b200.DeterministicRNG(132))
    sk = ctx.make_secret_key(tlwe_mask_size=2 if kind == 'k2' else 1)
    opts = {'compressed': {'compressed': True}, 'multi_bit': {'multi_bit': 2}, 'k2': {}}[kind]
    ck, cpk = ctx.make_cloud_key(sk, compact_public_key=True, **opts)
    if kind == 'compressed':
        ck = ck.decompress(ctx.thread)
    vm = ctx.make_virtual_machine(ck)
    B = 1100 if kind == 'k2' else 4096
    x, y = numpy.random.RandomState(5).randint(0, 2, (2, B)).astype(bool)
    cx = vm.expand(ctx.load_compact_ciphertext(ctx.encrypt(cpk, x).dumps()))
    cy = vm.expand(ctx.encrypt(cpk, y))
    if kind == 'k2':
        assert tuple(ctx.encrypt(cpk, x).data.shape) == (2, 3, N)
    assert (ctx.decrypt(sk, cx) == x).all()
    assert (ctx.decrypt(sk, vm.gate_nand(cx, cy)) == ~(x & y)).all()


def test_expansion_noise(api):
    """Phase error of 65 536 expanded samples under the secret key: sample variance within 0.5 - 2 times the DESIGN.md
    estimate (compact.noise_terms), nothing beyond 7 sigma."""
    nufhe, ctx, sk, ck, cpk, vm = api
    from nufhe_b200.lwe import lwe_decrypt
    from nufhe_b200.api_low_level import bool_to_t32
    bits = numpy.random.RandomState(7).randint(0, 2, 65536).astype(bool)
    out = vm.expand(ctx.encrypt(cpk, bits))
    err = compact_ref.i32(lwe_decrypt(ctx.thread, out, sk.lwe_key).astype(numpy.int64)
                          - bool_to_t32(bits).astype(numpy.int64)).astype(numpy.float64) * 2.0**-32
    est = sum(nufhe.compact.noise_terms(sk.params))
    var = float(err.var())
    print('compact expansion noise: measured variance %.4g, estimate %.4g (ratio %.3f), mean %.3g, max |err| %.2f sigma'
          % (var, est, var / est, err.mean(), numpy.abs(err).max() / est**0.5))
    assert 0.5 * est <= var <= 2 * est
    assert numpy.abs(err).max() <= 7 * est**0.5
    cv = out.current_variances.cpu().numpy()
    assert 0.9 * est <= cv.mean() <= 1.1 * est
    assert (ctx.decrypt(sk, out) == bits).all()
