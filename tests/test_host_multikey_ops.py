"""CPU tests of the multi-key tree LUTs, packing, expansion, index lookups and per-tenant LUT tables
(nufhe_b200/multikey.py, DESIGN.md section 18): the tile and group tables of csrc/mk_layout.cuh through the host
emulator, argument checks, and every operation equal per tenant to that tenant's own VirtualMachine on the engine
double."""
import ctypes
import os

import numpy
import pytest

import nufhe_b200
from nufhe_b200 import compact, index_lookup, packing, tree_lut
from nufhe_b200.random_numbers import DeterministicRNG
from multikey_ops_fake import MultiKeyOpsFakeEngine
import tree_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 1024


@pytest.fixture(scope='module')
def emul():
    path = os.path.join(ROOT, 'nufhe_b200', 'csrc', 'libnb_host_emul.so')
    if not os.path.exists(path):
        import __graft_entry__ as g
        g.build()
    lib = ctypes.CDLL(path)
    lib.emul_mk_tree_tiles.restype = ctypes.c_uint64
    lib.emul_mk_tree_tiles.argtypes = [ctypes.c_void_p, ctypes.c_size_t] + [ctypes.c_void_p] * 3
    lib.emul_mk_tree_keyswitch.restype = None
    lib.emul_mk_tree_keyswitch.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_size_t, ctypes.c_size_t, ctypes.c_int,
                                                                   ctypes.c_void_p]
    lib.emul_mk_group_tenants.restype = ctypes.c_uint64
    lib.emul_mk_group_tenants.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    lib.emul_pack_digits.restype = None
    lib.emul_pack_digits.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    return lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _sizes(counts):
    return numpy.asarray(counts, numpy.uintp)


def _tiles(emul, counts):
    c = _sizes(counts)
    n = emul.emul_mk_tree_tiles(_p(c), len(counts), None, None, None)
    row0, rows, tenant = numpy.zeros(n, numpy.uint64), numpy.zeros(n, numpy.uint32), numpy.zeros(n, numpy.uint32)
    assert emul.emul_mk_tree_tiles(_p(c), len(counts), _p(row0), _p(rows), _p(tenant)) == n
    return row0.astype(numpy.int64), rows.astype(numpy.int64), tenant.astype(numpy.int64)


# ---------------------------------------------------------------- tables (host emulator)

@pytest.mark.parametrize('counts', [(0,), (1,), (255,), (256,), (257,), (0, 1, 255, 256, 257, 0), (513, 2, 0, 700)])
def test_tree_tiles_never_cross_a_tenant_and_cover_every_row_once(emul, counts):
    row0, rows, tenant = _tiles(emul, counts)
    owner = numpy.repeat(numpy.arange(len(counts)), counts)
    covered = numpy.zeros(sum(counts), int)
    for r0, r, t in zip(row0, rows, tenant):
        assert 1 <= r <= 256
        assert (owner[r0:r0 + r] == t).all()
        covered[r0:r0 + r] += 1
    assert (covered == 1).all()
    assert len(row0) == sum(-(-c // 256) for c in counts)
    assert (numpy.diff(row0) > 0).all()


def test_tree_keyswitch_emulator_per_tenant_keys(emul):
    """Each tenant's rows of the emulated multi-key tree key switch equal tree_ref with that tenant's key."""
    rng = numpy.random.RandomState(5)
    n, k = 37, 1
    counts = [3, 0, 257, 1]
    keys = [(rng.randint(-2**31, 2**31, size=(n, 2, k, N), dtype=numpy.int64).astype(numpy.int32),
             rng.randint(-2**31, 2**31, size=(n, 2, N), dtype=numpy.int64).astype(numpy.int32)) for _ in counts]
    a = rng.randint(-2**31, 2**31, size=(sum(counts), n), dtype=numpy.int64).astype(numpy.int32)
    masks = (ctypes.c_void_p * len(counts))(*[m.ctypes.data for m, _ in keys])
    bodies = (ctypes.c_void_p * len(counts))(*[b.ctypes.data for _, b in keys])
    out = numpy.full((sum(counts), k + 1, N), 7, numpy.int32)
    emul.emul_mk_tree_keyswitch(_p(a), masks, bodies, _p(_sizes(counts)), len(counts), n, k, _p(out))
    lo = 0
    for t, c in enumerate(counts):
        if c:
            assert (out[lo:lo + c] == tree_ref.keyswitch(a[lo:lo + c], *keys[t])).all(), t
        lo += c


def test_pack_group_layout_and_zero_padding(emul):
    """The groups of mk.pack: tenant t owns ceil(B_t / N) consecutive groups; a zero padding row has the digits of an
    empty slot (0) and, with a zero body, the body coefficient of an empty slot (round_16(0 - C))."""
    counts = [1, 0, 1024, 1025, 3]
    groups = [-(-c // N) for c in counts]
    owner = numpy.zeros(sum(groups), numpy.uint32)
    assert emul.emul_mk_group_tenants(_p(_sizes(groups)), len(groups), _p(owner)) == sum(groups)
    assert list(owner) == [0, 2, 3, 3, 4]
    zero = numpy.zeros(64, numpy.int32)
    d = numpy.full(128, 9, numpy.int32)
    emul.emul_pack_digits(_p(zero), zero.size, _p(d))
    assert (d == 0).all()
    assert packing.PACK_LEVELS == 2


# ---------------------------------------------------------------- the Python layer on the engine double

@pytest.fixture(scope='module')
def env():
    ctx = nufhe_b200.Context(rng=DeterministicRNG(20261018), thread=MultiKeyOpsFakeEngine())
    sks, cks, tks, iks, cpks, pks, psks = [], [], [], [], [], [], []
    for _ in range(2):
        sk = ctx.make_secret_key()
        ck, tk, ik, cpk = ctx.make_cloud_key(sk, tree_key=True, index_key=True, compact_public_key=True)
        psk, pk = ctx.make_packing_keys(sk)
        for lst, v in zip((sks, cks, tks, iks, cpks, pks, psks), (sk, ck, tk, ik, cpk, pk, psk)):
            lst.append(v)
    # tenants: key 0, key 1, key 0 again (a repeated key), an idle tenant on key 1
    order = [0, 1, 0, 1]
    machine = ctx.make_multi_key_machine([cks[k] for k in order])
    vms = [ctx.make_virtual_machine(ck) for ck in cks]
    return dict(ctx=ctx, sks=sks, cks=cks, tks=tks, iks=iks, cpks=cpks, pks=pks, psks=psks, order=order,
                machine=machine, vms=vms)


def _same(x, y):
    return (tuple(x.shape) == tuple(y.shape) and (x.a == y.a).all() and (x.b == y.b).all()
            and (x.current_variances == y.current_variances).all())


def test_argument_checks(env):
    ctx, machine, order = env['ctx'], env['machine'], env['order']
    sks, tks, pks = env['sks'], env['tks'], env['pks']
    vm = env['vms'][0]
    x = ctx.encrypt_int(sks[0], [1], 2)
    xs = [x, None, None, None]
    table = vm.make_tree_lut(numpy.zeros((4, 4), int), bits=2, digits=2)
    with pytest.raises(ValueError, match='4 entries'):
        machine.lut_tree(tks[:1], table, [xs, xs])
    with pytest.raises(TypeError, match='tenant 0'):
        machine.lut_tree([None, tks[1], tks[0], None], table, [xs, xs])
    with pytest.raises(TypeError, match='tenant 0'):
        machine.lut_tree([pks[0], None, None, None], table, [xs, xs])
    with pytest.raises(ValueError, match='operand 1'):
        machine.lut_tree([tks[0]] * 4, table, [xs, xs[:2]])
    with pytest.raises(ValueError, match='takes 2 digits'):
        machine.lut_tree([tks[0]] * 4, table, [xs])
    other_ctx = nufhe_b200.Context(rng=DeterministicRNG(3), thread=ctx.thread)
    other_sk = other_ctx.make_secret_key(tlwe_mask_size=2)
    other_pk = other_ctx.make_packing_keys(other_sk)[1]
    with pytest.raises(ValueError, match='tenant 0'):
        machine.pack([other_pk, None, None, None], xs)
    with pytest.raises(TypeError, match='tenant 0'):
        machine.pack([tks[0], None, None, None], xs)
    with pytest.raises(ValueError, match='4 entries'):
        machine.pack(pks, xs)
    with pytest.raises(TypeError, match='tenant 2'):
        machine.expand([None, None, x, None])
    idx = ctx.encrypt_index(env['iks'][0], [1], 3)
    itab = vm.make_index_table(numpy.arange(8), bits=3)
    with pytest.raises(TypeError, match='tenant 1.*decompress'):
        machine.lookup([None, ctx.encrypt_index(env['iks'][1], [1], 3, compressed=True), None, None], itab)
    with pytest.raises(ValueError, match='tenant 0.*3-bit'):
        machine.lookup([ctx.encrypt_index(env['iks'][0], [1], 4), None, None, None], itab)
    with pytest.raises(ValueError, match='4 entries'):
        machine.lookup([idx], itab)
    # per-tenant LUT tables
    t2 = vm.make_lut([0, 1, 2, 3], bits=2)
    with pytest.raises(ValueError, match='tenant 2'):
        machine.lut([t2, None, vm.make_lut([0, 1, 0, 1, 0, 1, 0, 1], bits=3), None], [x, None, x, None])
    with pytest.raises(ValueError, match='tenant 2'):
        machine.lut([t2, None, vm.make_lut([0, 1, 1, 0], bits=2, out='bool'), None], [x, None, x, None])
    with pytest.raises(TypeError, match='tenant 2'):
        machine.lut([t2, None, None, None], [x, None, x, None])
    with pytest.raises(ValueError, match='one per tenant'):
        machine.lut([t2], [x, None, None, None])
    assert machine.lut([t2, None, None, None], [None] * 4) == [None] * 4


def test_lut_per_tenant_tables(env):
    ctx, machine, sks, vms, order = env['ctx'], env['machine'], env['sks'], env['vms'], env['order']
    fs = [lambda v: (v + 1) % 4, lambda v: 3 - v, lambda v: (v * v) % 4]
    tables = [vms[0].make_lut([f(v) for v in range(4)], bits=2) for f in fs] + [None]
    vals = [numpy.array([0, 3]), numpy.array([1]), numpy.array([[2, 1], [0, 3]]), None]
    xs = [None if v is None else ctx.encrypt_int(sks[order[t]], v, 2) for t, v in enumerate(vals)]
    out = machine.lut(tables, xs)
    assert out[3] is None
    for t in range(3):
        assert _same(out[t], vms[order[t]].lut(tables[t], xs[t])), t
        assert (ctx.decrypt_int(sks[order[t]], out[t], 2) == fs[t](vals[t])).all(), t


@pytest.mark.parametrize('bits,D', [(1, 2), (2, 2)])
def test_lut_tree(env, bits, D):
    ctx, machine, sks, vms, tks, order = (env[k] for k in ('ctx', 'machine', 'sks', 'vms', 'tks', 'order'))
    M = 1 << bits
    rng = numpy.random.RandomState(bits + 10 * D)
    tables = rng.randint(0, M, size=(2,) + (M,) * D)
    table = vms[0].make_tree_lut(tables, bits, D)
    sizes = [2, 1, 3, None]
    vals = [None if s is None else rng.randint(0, M, size=(D, s)) for s in sizes]
    digits = [[None if v is None else ctx.encrypt_int(sks[order[t]], v[i], bits) for t, v in enumerate(vals)]
              for i in range(D)]
    tree_keys = [tks[order[t]] for t in range(3)] + [None]
    out = machine.lut_tree(tree_keys, table, digits)
    assert out[3] is None
    for t in range(3):
        want = vms[order[t]].lut_tree(tks[order[t]], table, [d[t] for d in digits])
        assert len(out[t]) == 2 and all(_same(o, w) for o, w in zip(out[t], want)), t
        for f in range(2):
            truth = tables[(f,) + tuple(vals[t])]
            assert (ctx.decrypt_int(sks[order[t]], out[t][f], bits) == truth).all(), (t, f)


def test_lut_tree_pass_boundary(env, monkeypatch):
    """A pass of one ciphertext: tenants are cut between passes."""
    ctx, machine, sks, vms, tks, order = (env[k] for k in ('ctx', 'machine', 'sks', 'vms', 'tks', 'order'))
    table = vms[0].make_tree_lut(numpy.array([[0, 1], [1, 0]]), 1, 2, out='bool')
    monkeypatch.setattr(tree_lut, 'ROWS_PER_PASS', table.groups)
    vals = [numpy.array([[0, 1], [1, 1]]), numpy.array([[1], [0]]), None, None]
    digits = [[None if v is None else ctx.encrypt_int(sks[order[t]], v[i], 1) for t, v in enumerate(vals)]
              for i in range(2)]
    out = machine.lut_tree([tks[0], tks[1], None, None], table, digits)
    for t in range(2):
        assert _same(out[t], vms[order[t]].lut_tree(tks[order[t]], table, [d[t] for d in digits])), t
        assert (ctx.decrypt(sks[order[t]], out[t]) == (vals[t][0] ^ vals[t][1]).astype(bool)).all()


def test_pack(env):
    ctx, machine, sks, vms, pks, psks, order = (env[k] for k in ('ctx', 'machine', 'sks', 'vms', 'pks', 'psks', 'order'))
    bits = [numpy.array([True, False, True]), None, numpy.array([[False], [True]]), numpy.array([True])]
    cts = [None if b is None else ctx.encrypt(sks[order[t]], b) for t, b in enumerate(bits)]
    keys = [pks[order[t]] if b is not None else None for t, b in enumerate(bits)]
    out = machine.pack(keys, cts)
    assert out[1] is None
    for t in (0, 2, 3):
        assert out[t] == vms[order[t]].pack(pks[order[t]], cts[t]), t
        assert (ctx.decrypt(psks[order[t]], out[t]) == bits[t]).all(), t


def test_expand_with_pass_boundary(env, monkeypatch):
    ctx, machine, sks, vms, cpks, order = (env[k] for k in ('ctx', 'machine', 'sks', 'vms', 'cpks', 'order'))
    bits = [numpy.array([True, False]), numpy.array([[True], [True], [False]]), None, numpy.array([False])]
    cs = [None if b is None else ctx.encrypt(cpks[order[t]], b) for t, b in enumerate(bits)]
    for per_pass in (None, 1):
        if per_pass:
            monkeypatch.setattr(compact, 'groups_per_pass', lambda params: per_pass)
        out = machine.expand(cs)
        assert out[2] is None
        for t in (0, 1, 3):
            assert _same(out[t], vms[order[t]].expand(cs[t])), (per_pass, t)
            assert (ctx.decrypt(sks[order[t]], out[t]) == bits[t]).all()


@pytest.mark.parametrize('W', [1, 2])
def test_lookup_with_pass_boundary(env, monkeypatch, W):
    ctx, machine, sks, vms, iks, order = (env[k] for k in ('ctx', 'machine', 'sks', 'vms', 'iks', 'order'))
    m = 2
    rng = numpy.random.RandomState(W)
    entries = rng.randint(0, 4, size=(W, 1 << m))
    table = vms[0].make_index_table(entries if W > 1 else entries[0], bits=2)
    vals = [numpy.array([3, 0]), None, numpy.array([1]), numpy.array([[2]])]
    idx = [None if v is None else ctx.encrypt_index(iks[order[t]], v, m) for t, v in enumerate(vals)]
    for per_pass in (None, 1):
        if per_pass:
            monkeypatch.setattr(index_lookup, 'queries_per_pass', lambda m_, w_: per_pass)
        out = machine.lookup(idx, table)
        assert out[1] is None
        for t in (0, 2, 3):
            want = vms[order[t]].lookup(idx[t], table)
            got, want = ([out[t]], [want]) if W == 1 else (out[t], want)
            assert len(got) == W and all(_same(g, w) for g, w in zip(got, want)), (per_pass, t)
            for w in range(W):
                assert (ctx.decrypt_int(sks[order[t]], got[w], 2) == entries[w][vals[t]]).all(), (t, w)


def test_dest(env):
    """lut_tree and lookup write into `dest` when it is given."""
    ctx, machine, sks, vms, tks, iks, order = (env[k] for k in ('ctx', 'machine', 'sks', 'vms', 'tks', 'iks', 'order'))
    table = vms[0].make_tree_lut(numpy.array([[0, 1], [1, 1]]), 1, 2, out='bool')
    vals = [numpy.array([[0, 1], [0, 0]]), None, None, numpy.array([[1], [0]])]
    digits = [[None if v is None else ctx.encrypt_int(sks[order[t]], v[i], 1) for t, v in enumerate(vals)]
              for i in range(2)]
    dest = [None if v is None else machine.empty_ciphertext(v[0].shape) for v in vals]
    with pytest.raises(ValueError, match='tenant 1'):
        machine.lut_tree([tks[0], tks[1], None, tks[1]], table, digits, dest=[dest[0], dest[0], None, dest[3]])
    out = machine.lut_tree([tks[0], None, None, tks[1]], table, digits, dest=dest)
    for t in (0, 3):
        assert out[t] is dest[t]
        assert _same(out[t], vms[order[t]].lut_tree(tks[order[t]], table, [d[t] for d in digits])), t
    itab = vms[0].make_index_table(numpy.array([[0, 1, 2, 3], [3, 2, 1, 0]]), bits=2)
    idx = [ctx.encrypt_index(iks[0], [2, 1], 2), None, None, None]
    dest = [[machine.empty_ciphertext((2,)) for _ in range(2)], None, None, None]
    out = machine.lookup(idx, itab, dest=dest)
    assert out[0][0] is dest[0][0] and out[0][1] is dest[0][1]
    want = vms[0].lookup(idx[0], itab)
    assert all(_same(g, w) for g, w in zip(out[0], want))
