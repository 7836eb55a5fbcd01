"""The multi-key machine on compressed cloud keys (resident_tenants, DESIGN.md section 19) on the GPU.

Through the C ABI, inside sentinel guards: nb_mk_bk_expand writes, for several tenants in one launch, exactly the FP64
part that nb_bk_prepare stores for the decompressed key and nothing else; nb_mk_ks_expand writes exactly decompress()'s
ks_a; both refuse null pointers and other shapes, and a released slot is no longer a key.  Through Python, every
operation of the machine with R = 1, 3 and 6 on real compressed keys equals each tenant's own VirtualMachine on the
decompressed key and decrypts to the truth table; 600 synthetic tenants at R = 64 run in rounds and match their
decompressed keys on both sides of every round boundary."""
import ctypes

import numpy
import pytest
import torch

pytestmark = pytest.mark.gpu
N = 1024
GUARD = 4096
SENTINEL = 0x5a5a5a5a5a5a5a5a


@pytest.fixture(scope='module')
def eng():
    from nufhe_b200.engine import Engine
    return Engine(0)


@pytest.fixture(scope='module')
def params():
    from nufhe_b200.api_low_level import NuFHEParameters
    return NuFHEParameters()


def rand_i32(rng, shape):
    return rng.randint(-2**31, 2**31, size=shape, dtype=numpy.int64).astype(numpy.int32)


def synthetic_key(eng, params, rng):
    """A CompressedCloudKey with a random seed and random bodies on the device (no secret key behind it)."""
    from nufhe_b200.compressed import CompressedCloudKey
    n = params.in_out_params.size
    seed = rng.randint(0, 2**32, size=8, dtype=numpy.int64).astype(numpy.uint32)
    body = eng.to_device(rand_i32(rng, (n, 2, 2, N)))
    ks_b = eng.to_device(rand_i32(rng, (1024, params.ks_decomp_length, 1 << params.ks_log2_base)))
    return CompressedCloudKey(params, seed, body, 1e-9, ks_b, 2e-9)


def decompressed_fp64(eng, key):
    from nufhe_b200.tgsw import engine_format
    bk = engine_format(eng, key.decompress(eng).bootstrap_key.tgsw)
    return bk[:, _ntt_u64(eng):].cpu().numpy()


def _ntt_u64(eng):
    return eng.lib.nb_bk_row_u64() - eng.lib.nb_bk_multibit_row_u64()


def test_bk_expand_is_word_identical_to_bk_prepare(eng, params):
    rng = numpy.random.RandomState(19)
    n, row = params.in_out_params.size, eng.lib.nb_bk_row_u64()
    keys = [synthetic_key(eng, params, rng) for _ in range(2)]
    # extreme bodies: every coefficient of one polynomial at -2^31, of another at 2^31 - 1
    keys[0].bk_body[0, 0, 0].fill_(-2**31)
    keys[0].bk_body[n - 1, 1, 1].fill_(2**31 - 1)
    keys[1].bk_body[7, 1, 0].fill_(-2**31)
    tenants = [keys[0], keys[1], keys[0]]                  # one tenant repeated, into its own slot
    buf = torch.full((len(tenants) * (n * row + GUARD) + GUARD,), SENTINEL, dtype=torch.int64, device=eng.device)
    slots = [buf[GUARD + i * (n * row + GUARD):][:n * row].view(n, row) for i in range(len(tenants))]
    eng.mk_bk_expand(numpy.stack([k.seed for k in tenants]), [k.bk_body for k in tenants], slots, params)
    h = buf.cpu().numpy()
    ntt = _ntt_u64(eng)
    for i, key in enumerate(tenants):
        lo = GUARD + i * (n * row + GUARD)
        assert (h[lo - GUARD:lo] == SENTINEL).all(), 'a store before slot %d' % i
        got = h[lo:lo + n * row].reshape(n, row)
        assert (got[:, :ntt] == SENTINEL).all(), 'a store into the NTT planes of slot %d' % i
        assert (got[:, ntt:] == decompressed_fp64(eng, key)).all(), 'slot %d' % i
    assert (h[-GUARD:] == SENTINEL).all()
    for s in slots:
        eng.lib.nb_mk_slot_release(eng.handle, ctypes.c_void_p(s.data_ptr()))


def test_ks_expand_is_decompress(eng, params):
    rng = numpy.random.RandomState(23)
    keys = [synthetic_key(eng, params, rng) for _ in range(2)]
    shape = (1024, params.ks_decomp_length, 1 << params.ks_log2_base, params.in_out_params.size)
    size = int(numpy.prod(shape))
    fill = 0x3c3c3c3c
    buf = torch.full((2 * (size + GUARD) + GUARD,), fill, dtype=torch.int32, device=eng.device)
    ks_as = [buf[GUARD + i * (size + GUARD):][:size].view(shape) for i in range(2)]
    eng.mk_ks_expand(numpy.stack([k.seed for k in keys]), ks_as)
    h = buf.cpu().numpy()
    for i, key in enumerate(keys):
        lo = GUARD + i * (size + GUARD)
        assert (h[lo - GUARD:lo] == fill).all()
        want = key.decompress(eng).keyswitch_key.lwe.a.cpu().numpy()
        assert (h[lo:lo + size].reshape(shape) == want).all(), i
    assert (h[-GUARD:] == fill).all()


def test_expand_calls_refuse_bad_arguments(eng, params):
    from nufhe_b200 import _native as nv
    lib, h = eng.lib, eng.handle
    n = params.in_out_params.size
    seeds = (ctypes.c_uint32 * 8)()
    slot = eng.mk_bk_slot(n)
    body = torch.zeros((n, 2, 2, N), dtype=torch.int32, device=eng.device)
    ks_a = torch.zeros((1024, 8, 4, n), dtype=torch.int32, device=eng.device)
    vp = ctypes.c_void_p
    one = lambda x: (vp * 1)(x.data_ptr())
    null = (vp * 1)(None)
    # zero tenants: a no-op
    assert lib.nb_mk_bk_expand(h, None, None, None, 0, n, 1, 2, N) == nv.NB_OK
    assert lib.nb_mk_ks_expand(h, None, None, 0, 1024, 8, 2, n) == nv.NB_OK
    # null pointers
    assert lib.nb_mk_bk_expand(h, None, one(body), one(slot), 1, n, 1, 2, N) == nv.NB_EINVAL
    assert lib.nb_mk_bk_expand(h, seeds, null, one(slot), 1, n, 1, 2, N) == nv.NB_EINVAL
    assert lib.nb_mk_bk_expand(h, seeds, one(body), null, 1, n, 1, 2, N) == nv.NB_EINVAL
    assert lib.nb_mk_ks_expand(h, None, one(ks_a), 1, 1024, 8, 2, n) == nv.NB_EINVAL
    assert lib.nb_mk_ks_expand(h, seeds, null, 1, 1024, 8, 2, n) == nv.NB_EINVAL
    assert lib.nb_mk_slot_release(h, None) == nv.NB_EINVAL
    # other shapes
    for k, l, big_n, nn in ((2, 2, N, n), (1, 3, N, n), (1, 2, 2048, n), (1, 2, N, 0), (1, 2, N, 1025)):
        assert lib.nb_mk_bk_expand(h, seeds, one(body), one(slot), 1, nn, k, l, big_n) == nv.NB_EUNSUPPORTED
    for in_size, t, lb, nn in ((512, 8, 2, n), (1024, 7, 2, n), (1024, 8, 3, n), (1024, 8, 2, 630)):
        assert lib.nb_mk_ks_expand(h, seeds, one(ks_a), 1, in_size, t, lb, nn) == nv.NB_EUNSUPPORTED
    eng.synchronize()


def test_released_slot_is_no_key(eng, params):
    from nufhe_b200.gates import MU
    rng = numpy.random.RandomState(29)
    n = params.in_out_params.size
    key = synthetic_key(eng, params, rng)
    slot = eng.mk_bk_slot(n)
    empty = (eng.empty((0, n), torch.int32), eng.empty((0,), torch.int32))
    eng.mk_bk_expand(key.seed[None], [key.bk_body], [slot], params)
    eng.mk_bootstrap_extract(empty, None, 0, 1, 0, MU, [slot], [0])
    eng.lib.nb_mk_slot_release(eng.handle, ctypes.c_void_p(slot.data_ptr()))
    # the key check runs before the empty batch returns, so nothing is read
    with pytest.raises(ValueError, match='not inside'):
        eng.mk_bootstrap_extract(empty, None, 0, 1, 0, MU, [slot], [0])


# ---------------------------------------------------------------- the machine on real compressed keys

@pytest.fixture(scope='module')
def real():
    import nufhe_b200
    ctx = nufhe_b200.Context(rng=nufhe_b200.DeterministicRNG(20261018))
    sks, cks, tks, iks, cpks = [], [], [], [], []
    for _ in range(6):
        sk = ctx.make_secret_key()
        ck, tk, ik, cpk = ctx.make_cloud_key(sk, compressed=True, tree_key=True, index_key=True,
                                             compact_public_key=True)
        for lst, v in zip((sks, cks, tks, iks, cpks), (sk, ck, tk, ik, cpk)):
            lst.append(v)
    cks = [ctx.load_compressed_cloud_key(ck.dumps()) for ck in cks]
    vms = [ctx.make_virtual_machine(ck.decompress(ctx.thread)) for ck in cks]
    return dict(ctx=ctx, sks=sks, cks=cks, tks=tks, iks=iks, cpks=cpks, vms=vms)


def _same(x, y):
    return (tuple(x.shape) == tuple(y.shape) and torch.equal(x.a, y.a) and torch.equal(x.b, y.b)
            and torch.equal(x.current_variances, y.current_variances))


@pytest.mark.parametrize('R', [1, 3, 6])
def test_machine_every_operation(real, R):
    ctx, sks, cks, tks, iks, cpks, vms = (real[k] for k in ('ctx', 'sks', 'cks', 'tks', 'iks', 'cpks', 'vms'))
    T = len(cks)
    m = ctx.make_multi_key_machine(cks, resident_tenants=R)
    rng = numpy.random.RandomState(R)
    active = [0, 1, 2, 4, 5]                                # tenant 3 idle
    bits = [rng.randint(0, 2, size=(3, 4)).astype(bool) if t in active else None for t in range(T)]
    xs = [[None if b is None else ctx.encrypt(sks[t], b[i]) for t, b in enumerate(bits)] for i in range(3)]
    for name, f in (('nand', lambda a, b: ~(a & b)), ('xor', lambda a, b: a ^ b)):
        out = getattr(m, 'gate_' + name)(xs[0], xs[1])
        assert out[3] is None and len(m.resident) == min(R, len(active))
        for t in active:
            assert _same(out[t], getattr(vms[t], 'gate_' + name)(xs[0][t], xs[1][t])), (name, t)
            assert (ctx.decrypt(sks[t], out[t]) == f(bits[t][0], bits[t][1])).all(), (name, t)
    dest = [None if b is None else m.empty_ciphertext((4,)) for b in bits]
    out = m.gate_mux(xs[0], xs[1], xs[2], dest=dest)
    for t in active:
        assert out[t] is dest[t] and _same(out[t], vms[t].gate_mux(xs[0][t], xs[1][t], xs[2][t])), t
        assert (ctx.decrypt(sks[t], out[t]) == numpy.where(bits[t][0], bits[t][1], bits[t][2])).all()
    # per-tenant tables with 2 outputs
    fs = [(lambda v, s=s: (v + s) % 4, lambda v, s=s: (3 * v + s) % 4) for s in range(T)]
    tables = [vms[0].make_lut([[g(v) for v in range(4)] for g in fs[t]], bits=2) if t in active else None
              for t in range(T)]
    vals = [rng.randint(0, 4, size=3) if t in active else None for t in range(T)]
    ys = [None if v is None else ctx.encrypt_int(sks[t], v, 2) for t, v in enumerate(vals)]
    out = m.lut(tables, ys)
    for t in active:
        want = vms[t].lut(tables[t], ys[t])
        assert all(_same(o, w) for o, w in zip(out[t], want)), t
        for o, g in zip(out[t], fs[t]):
            assert (ctx.decrypt_int(sks[t], o, 2) == g(vals[t])).all(), t
    # tree LUT on two 2-bit digits
    tt = rng.randint(0, 4, size=(4, 4))
    table = vms[0].make_tree_lut(tt, 2, 2)
    dv = [rng.randint(0, 4, size=(2, 2)) if t in active else None for t in range(T)]
    digits = [[None if v is None else ctx.encrypt_int(sks[t], v[i], 2) for t, v in enumerate(dv)] for i in range(2)]
    out = m.lut_tree([tks[t] if t in active else None for t in range(T)], table, digits)
    for t in active:
        assert _same(out[t], vms[t].lut_tree(tks[t], table, [d[t] for d in digits])), t
        assert (ctx.decrypt_int(sks[t], out[t], 2) == tt[tuple(dv[t])]).all(), t
    # compact expansion and index lookups
    cs = [None if b is None else ctx.encrypt(cpks[t], b[0]) for t, b in enumerate(bits)]
    out = m.expand(cs)
    for t in active:
        assert _same(out[t], vms[t].expand(cs[t])) and (ctx.decrypt(sks[t], out[t]) == bits[t][0]).all(), t
    entries = rng.randint(0, 4, size=8)
    itab = vms[0].make_index_table(entries, bits=3)         # 3-bit entries, 3-bit indices
    iv = [rng.randint(0, 8, size=2) if t in active else None for t in range(T)]
    idx = [None if v is None else ctx.encrypt_index(iks[t], v, 3) for t, v in enumerate(iv)]
    out = m.lookup(idx, itab)
    for t in active:
        assert _same(out[t], vms[t].lookup(idx[t], itab)), t
        assert (ctx.decrypt_int(sks[t], out[t], 3) == entries[iv[t]]).all(), t


def test_one_slot_refilled_again_and_again(real):
    ctx, sks, cks, vms = (real[k] for k in ('ctx', 'sks', 'cks', 'vms'))
    m = ctx.make_multi_key_machine(cks, resident_tenants=1)
    T = len(cks)
    for step in range(6):
        t = step % 2
        x = ctx.encrypt(sks[t], [True, False, step % 3 == 0])
        ops = [x if u == t else None for u in range(T)]
        out = m.gate_nand(ops, ops)
        assert m.resident == [t]
        assert _same(out[t], vms[t].gate_nand(x, x)), step
        assert (ctx.decrypt(sks[t], out[t]) == ~numpy.array([True, False, step % 3 == 0])).all()


def test_600_tenants_at_64_resident(eng, params):
    """More tenants than 80 GB could hold resident (250 MB each): one NAND each in rounds of 64."""
    import nufhe_b200
    ctx = nufhe_b200.Context(rng=nufhe_b200.DeterministicRNG(7))
    thr = ctx.thread
    rng = numpy.random.RandomState(31)
    T, R = 600, 64
    keys = [synthetic_key(thr, params, rng) for _ in range(T)]
    m = ctx.make_multi_key_machine(keys, resident_tenants=R)
    n = params.in_out_params.size
    from nufhe_b200.lwe import LweSampleArray
    cv = lambda: torch.zeros((1,), dtype=torch.float32, device=thr.device)
    xs = [LweSampleArray(params.in_out_params, thr.to_device(rand_i32(rng, (1, n))), thr.to_device(rand_i32(rng, (1,))),
                         cv()) for _ in range(T)]
    ys = [LweSampleArray(params.in_out_params, thr.to_device(rand_i32(rng, (1, n))), thr.to_device(rand_i32(rng, (1,))),
                         cv()) for _ in range(T)]
    out = m.gate_nand(xs, ys)
    assert m.resident == list(range(T - R, T))
    sample = {0, T - 1} | {b for r in range(R, T, R) for b in (r - 1, r)}
    assert len(sample) >= 16
    for t in sorted(sample):
        vm = ctx.make_virtual_machine(keys[t].decompress(thr))
        assert _same(out[t], vm.gate_nand(xs[t], ys[t])), t
        del vm
