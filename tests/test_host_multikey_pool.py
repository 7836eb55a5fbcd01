"""CPU tests of the multi-key machine on compressed cloud keys (resident_tenants, DESIGN.md section 19): the index
arithmetic of csrc/mk_expand_layout.cuh through the host emulator against the ChaCha20 reference and NumPy, and the
machine with R = 1, 2 and T resident tenants on the engine double, every operation equal per tenant to that tenant's own
VirtualMachine on the decompressed key, with the round order, the LRU order and the refusals."""
import ctypes
import os

import numpy
import pytest

import nufhe_b200
from nufhe_b200.random_numbers import DeterministicRNG
from chacha_ref import chacha20_words, seeded_uniform
from multikey_pool_fake import MultiKeyPoolFakeEngine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 1024


@pytest.fixture(scope='module')
def emul():
    path = os.path.join(ROOT, 'nufhe_b200', 'csrc', 'libnb_host_emul.so')
    if not os.path.exists(path):
        import __graft_entry__ as g
        g.build()
    lib = ctypes.CDLL(path)
    u32, u64 = ctypes.c_uint32, ctypes.c_uint64
    lib.emul_mk_bk_mask_word.restype = u64
    lib.emul_mk_bk_mask_word.argtypes = [u64] + [u32] * 6
    lib.emul_mk_bk_body_offset.restype = u64
    lib.emul_mk_bk_body_offset.argtypes = [u64] + [u32] * 5
    lib.emul_mk_bk_mask_regroup.restype = None
    lib.emul_mk_bk_mask_regroup.argtypes = [ctypes.c_void_p, u64] + [u32] * 5 + [ctypes.c_void_p]
    lib.emul_mk_ks_expand.restype = None
    lib.emul_mk_ks_expand.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_int, ctypes.c_size_t,
                                      ctypes.c_void_p]
    return lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


SEED = numpy.array([0x01234567, 0x89abcdef, 0xdeadbeef, 0, 0xffffffff, 7, 1 << 31, 12345], numpy.uint32)


# ---------------------------------------------------------------- index arithmetic (host emulator)

@pytest.mark.parametrize('n,k,l', [(500, 1, 2), (3, 2, 3)])
def test_bk_mask_and_body_offsets(emul, n, k, l):
    """Mask polynomial (i, mi, j, mo) starts at its C-order index in (n, k+1, l, k, N); body (i, mi, j) at its index in
    (n, k+1, l, N): first and last rows, and mi, j and mo at their extremes."""
    for i in (0, 1, n - 1):
        for mi in (0, k):
            for j in (0, l - 1):
                for mo in (0, k - 1):
                    want = numpy.ravel_multi_index((i, mi, j, mo, 0), (n, k + 1, l, k, N))
                    assert emul.emul_mk_bk_mask_word(i, mi, j, mo, k, l, N) == want, (i, mi, j, mo)
                want = numpy.ravel_multi_index((i, mi, j, 0), (n, k + 1, l, N))
                assert emul.emul_mk_bk_body_offset(i, mi, j, k, l, N) == want, (i, mi, j)


@pytest.mark.parametrize('i,mi,j', [(0, 0, 0), (0, 1, 1), (1, 0, 1), (499, 1, 1), (499, 0, 0)])
def test_bk_mask_regroup_into_stride_64_order(emul, i, mi, j):
    """After the regrouping, thread n0 holds the mask coefficients 64 jj + n0 (bk_spectra_kernel's order) of the
    stream (seed, nonce 1)."""
    got = numpy.empty((64, 16), numpy.int32)
    emul.emul_mk_bk_mask_regroup(_p(SEED), i, mi, j, 0, 1, 2, _p(got))
    first = int(numpy.ravel_multi_index((i, mi, j, 0, 0), (500, 2, 2, 1, N)))
    words = chacha20_words(SEED, 1, first, N)
    assert (got == words.reshape(16, 64).T).all()


@pytest.mark.parametrize('in_size,t,log2_base,n', [(3, 2, 2, 7), (2, 3, 3, 5), (4, 8, 2, 500)])
def test_ks_a_rows_skip_h0(emul, in_size, t, log2_base, n):
    """The stream (seed, nonce 2) fills rows h >= 1 of ks_a in order and rows h = 0 are zero: decompress()'s ks_a."""
    base = 1 << log2_base
    got = numpy.full((in_size, t, base, n), 7, numpy.int32)
    emul.emul_mk_ks_expand(_p(SEED), in_size, t, log2_base, n, _p(got))
    want = numpy.zeros((in_size, t, base, n), numpy.int32)
    want[:, :, 1:, :] = seeded_uniform(SEED, 2, (in_size, t, base - 1, n))
    assert (got == want).all()


# ---------------------------------------------------------------- the machine on the engine double

@pytest.fixture(scope='module')
def env():
    thr = MultiKeyPoolFakeEngine()
    ctx = nufhe_b200.Context(rng=DeterministicRNG(20261018), thread=thr)
    sks, cks, tks, iks, cpks = [], [], [], [], []
    for _ in range(3):
        sk = ctx.make_secret_key()
        ck, tk, ik, cpk = ctx.make_cloud_key(sk, compressed=True, tree_key=True, index_key=True,
                                             compact_public_key=True)
        for lst, v in zip((sks, cks, tks, iks, cpks), (sk, ck, tk, ik, cpk)):
            lst.append(v)
    # tenants: keys 0, 1, 0 (a repeated key), 2; tests keep some idle
    order = [0, 1, 0, 2]
    vms = [ctx.make_virtual_machine(ck.decompress(thr)) for ck in cks]
    return dict(ctx=ctx, thr=thr, sks=sks, cks=cks, tks=tks, iks=iks, cpks=cpks, order=order, vms=vms)


def _machine(env, R):
    m = env['ctx'].make_multi_key_machine([env['cks'][k] for k in env['order']], resident_tenants=R)
    fill = m._pool.fill

    def checked_fill(machine, tenants):
        before = dict(m._pool.lru)
        fill(machine, tenants)
        # every tenant of the round holds a slot, and a slot it held before the round is the one it holds now
        for t in tenants:
            assert t in m._pool.lru, (t, tenants)
            if t in before:
                assert m._pool.lru[t] is before[t], (t, tenants)
    m._pool.fill = checked_fill
    return m


def _model(resident, active, R):
    """The documented order of `resident` after a call on `active` tenants."""
    lru = list(resident)
    order = [t for t in active if t in lru] + [t for t in active if t not in lru]
    for r0 in range(0, len(order), R):
        rnd = order[r0:r0 + R]
        victims = [t for t in lru if t not in rnd]
        for t in rnd:
            if t not in lru:
                if len(lru) == R:
                    lru.remove(victims.pop(0))
                lru.append(t)
        lru = [t for t in lru if t not in rnd] + sorted(rnd)
    return lru


def _same(x, y):
    return (tuple(x.shape) == tuple(y.shape) and (x.a == y.a).all() and (x.b == y.b).all()
            and (x.current_variances == y.current_variances).all())


RS = [1, 2, 4]


@pytest.mark.parametrize('R', RS)
def test_gates(env, R):
    ctx, sks, vms, order = env['ctx'], env['sks'], env['vms'], env['order']
    m = _machine(env, R)
    rng = numpy.random.RandomState(R)
    bits = [rng.randint(0, 2, size=(3, 2)).astype(bool) for _ in range(4)]
    bits[2] = None                                    # an idle tenant
    xs = [[None if b is None else ctx.encrypt(sks[order[t]], b[i]) for t, b in enumerate(bits)] for i in range(3)]
    active = [0, 1, 3]
    resident = []
    for name, f in (('nand', lambda a, b: ~(a & b)), ('xor', lambda a, b: a ^ b)):
        out = getattr(m, 'gate_' + name)(xs[0], xs[1])
        resident = _model(resident, active, R)
        assert m.resident == resident, name
        assert out[2] is None
        for t in active:
            want = getattr(vms[order[t]], 'gate_' + name)(xs[0][t], xs[1][t])
            assert _same(out[t], want), (name, t)
            assert (ctx.decrypt(sks[order[t]], out[t]) == f(bits[t][0], bits[t][1])).all()
    dest = [None if b is None else m.empty_ciphertext((2,)) for b in bits]
    out = m.gate_mux(xs[0], xs[1], xs[2], dest=dest)
    resident = _model(resident, active, R)
    assert m.resident == resident
    for t in active:
        assert out[t] is dest[t]
        assert _same(out[t], vms[order[t]].gate_mux(xs[0][t], xs[1][t], xs[2][t])), t
        assert (ctx.decrypt(sks[order[t]], out[t]) == numpy.where(bits[t][0], bits[t][1], bits[t][2])).all()
    # key-less gates expand nothing
    before = len(env['thr'].expansions)
    out = m.gate_not(xs[0])
    assert len(env['thr'].expansions) == before and m.resident == resident
    assert (ctx.decrypt(sks[order[1]], out[1]) == ~bits[1][0]).all()


def test_round_order_and_eviction(env):
    """R = 2 over 3 active tenants: rounds [0, 1], [2]; then the resident tenants [1, 2] first, [0] after, evicting the
    least recently used tenant outside the round each time; each round fills its slots with one launch per key part."""
    ctx, sks, order, thr = env['ctx'], env['sks'], env['order'], env['thr']
    m = _machine(env, 2)
    x = [ctx.encrypt(sks[order[t]], [True]) for t in range(3)] + [None]
    thr.expansions.clear()
    m.gate_nand(x, x)
    assert m.resident == [1, 2]
    assert thr.expansions == [('bk', 2), ('ks', 2), ('bk', 1), ('ks', 1)]
    m.gate_and(x, x)
    assert m.resident == [2, 0]
    assert thr.expansions[4:] == [('bk', 1), ('ks', 1)]
    # a call on resident tenants only expands nothing
    m.gate_or([None, None, x[2], None], [None, None, x[2], None])
    assert m.resident == [0, 2] and len(thr.expansions) == 6
    # a round of a resident tenant (the least recently used) and a new one evicts the tenant outside the round
    y = [x[0], None, None, ctx.encrypt(sks[order[3]], [False])]
    out = m.gate_nand(y, y)
    assert m.resident == [0, 3] and thr.expansions[6:] == [('bk', 1), ('ks', 1)]
    assert (ctx.decrypt(sks[order[3]], out[3]) == [True]).all()


@pytest.mark.parametrize('R', RS)
def test_lut_per_tenant_tables_two_outputs(env, R):
    ctx, sks, vms, order = env['ctx'], env['sks'], env['vms'], env['order']
    m = _machine(env, R)
    fs = [[lambda v: (v + 1) % 4, lambda v: 3 - v], [lambda v: v, lambda v: (v * v) % 4],
          [lambda v: 0 * v, lambda v: (v + 2) % 4], None]
    tables = [None if f is None else vms[0].make_lut([[g(v) for v in range(4)] for g in f], bits=2) for f in fs]
    vals = [numpy.array([0, 3]), numpy.array([1]), numpy.array([[2, 1]]), None]
    xs = [None if v is None else ctx.encrypt_int(sks[order[t]], v, 2) for t, v in enumerate(vals)]
    out = m.lut(tables, xs)
    assert out[3] is None and m.resident == _model([], [0, 1, 2], R)
    for t in range(3):
        want = vms[order[t]].lut(tables[t], xs[t])
        assert len(out[t]) == 2 and all(_same(o, w) for o, w in zip(out[t], want)), t
        for o, g in zip(out[t], fs[t]):
            assert (ctx.decrypt_int(sks[order[t]], o, 2) == g(vals[t])).all(), t


@pytest.mark.parametrize('R', RS)
def test_lut_tree(env, R):
    ctx, sks, vms, tks, order = (env[k] for k in ('ctx', 'sks', 'vms', 'tks', 'order'))
    m = _machine(env, R)
    rng = numpy.random.RandomState(R + 7)
    tables = rng.randint(0, 2, size=(2, 2))
    table = vms[0].make_tree_lut(tables, 1, 2)
    vals = [rng.randint(0, 2, size=(2, 2)), None, rng.randint(0, 2, size=(2, 1)), rng.randint(0, 2, size=(2, 1))]
    digits = [[None if v is None else ctx.encrypt_int(sks[order[t]], v[i], 1) for t, v in enumerate(vals)]
              for i in range(2)]
    tree_keys = [None if v is None else tks[order[t]] for t, v in enumerate(vals)]
    out = m.lut_tree(tree_keys, table, digits)
    assert out[1] is None and m.resident == _model([], [0, 2, 3], R)
    for t in (0, 2, 3):
        assert _same(out[t], vms[order[t]].lut_tree(tks[order[t]], table, [d[t] for d in digits])), t
        assert (ctx.decrypt_int(sks[order[t]], out[t], 1) == tables[tuple(vals[t])]).all(), t


@pytest.mark.parametrize('R', RS)
def test_expand_and_lookup(env, R):
    ctx, sks, vms, cpks, iks, order = (env[k] for k in ('ctx', 'sks', 'vms', 'cpks', 'iks', 'order'))
    m = _machine(env, R)
    bits = [numpy.array([True, False]), None, numpy.array([[True], [False]]), numpy.array([False])]
    cs = [None if b is None else ctx.encrypt(cpks[order[t]], b) for t, b in enumerate(bits)]
    out = m.expand(cs)
    assert out[1] is None and m.resident == _model([], [0, 2, 3], R)
    for t in (0, 2, 3):
        assert _same(out[t], vms[order[t]].expand(cs[t])), t
        assert (ctx.decrypt(sks[order[t]], out[t]) == bits[t]).all()
    entries = numpy.array([3, 1, 0, 2])
    table = vms[0].make_index_table(entries, bits=2)
    vals = [numpy.array([3, 0]), numpy.array([1]), None, numpy.array([[2]])]
    idx = [None if v is None else ctx.encrypt_index(iks[order[t]], v, 2) for t, v in enumerate(vals)]
    resident = m.resident
    out = m.lookup(idx, table)
    assert out[2] is None and m.resident == _model(resident, [0, 1, 3], R)
    for t in (0, 1, 3):
        assert _same(out[t], vms[order[t]].lookup(idx[t], table)), t
        assert (ctx.decrypt_int(sks[order[t]], out[t], 2) == entries[vals[t]]).all()


def test_refusals(env):
    ctx, cks, sks = env['ctx'], env['cks'], env['sks']
    thr = env['thr']
    decompressed = cks[0].decompress(thr)
    with pytest.raises(TypeError, match='tenant 1.*CompressedCloudKey'):
        ctx.make_multi_key_machine([cks[0], decompressed], resident_tenants=2)
    with pytest.raises(TypeError, match='tenant 0'):
        ctx.make_multi_key_machine(['not a key'], resident_tenants=2)
    with pytest.raises(ValueError, match='at least 1'):
        ctx.make_multi_key_machine(cks, resident_tenants=0)
    with pytest.raises(TypeError, match='int'):
        ctx.make_multi_key_machine(cks, resident_tenants=2.0)
    # without resident_tenants a compressed key is refused as before
    with pytest.raises(TypeError, match='tenant 0.*decompress'):
        ctx.make_multi_key_machine(cks)
    other_ctx = nufhe_b200.Context(rng=DeterministicRNG(3), thread=thr)
    other = other_ctx.make_cloud_key(other_ctx.make_secret_key(tlwe_mask_size=2), compressed=True)
    with pytest.raises(ValueError, match='tenant 1'):
        ctx.make_multi_key_machine([cks[0], other], resident_tenants=2)
    with pytest.raises(ValueError, match='tenant 0.*tlwe_mask_size=1'):
        ctx.make_multi_key_machine([other], resident_tenants=2)
    mb = ctx.make_cloud_key(sks[0], compressed=True, multi_bit=2)
    with pytest.raises(ValueError, match='tenant 1.*multi-bit'):
        ctx.make_multi_key_machine([cks[0], mb], resident_tenants=1)
