"""CPU tests of oblivious writes (nufhe_b200/index_write.py, DESIGN.md section 21): the oracle-composed write
(tests/write_ref.py) against the plain arithmetic it stands for, and the Python layer on the oracle-backed engine double
(scatter_add, write, argument errors, the noise rule, pickles of written tables, per-tenant writes on the multi-key
machine)."""
import numpy
import pytest
import torch

import nufhe_b200
from nufhe_b200 import index_lookup as IL
from nufhe_b200 import index_write, lut
from nufhe_b200.random_numbers import DeterministicRNG
from index_write_fake import IndexWriteFakeEngine
import index_ref as R
import write_ref as WR

N = 1024


@pytest.mark.parametrize('m, W', [(1, 1), (1, 3), (4, 3), (9, 2), (10, 1), (10, 2), (11, 1), (11, 2), (13, 1)])
def test_reference_adds_one_hot(m, W):
    """trivial selectors b H and values that are multiples of 2^12 (so that the rounded decomposition is exact): the
    write returns exactly table + onehot(idx) v, repeated indexes adding up"""
    rng = numpy.random.RandomState(m * 7 + W)
    P = IL.table_polys_count(m, W)
    table = (rng.randint(0, 2**20, size=(P, 2, N)).astype(numpy.int64) << 12).astype(numpy.uint32).view(numpy.int32)
    idx = numpy.concatenate([[0, (1 << m) - 1, 0], rng.randint(0, 1 << m, size=3)])
    Q = idx.size
    b = (rng.randint(0, 2**20, size=(Q, W)).astype(numpy.int64) << 12).astype(numpy.uint32).view(numpy.int32)
    bits = (idx[:, None] >> numpy.arange(m)) & 1
    sel = R.noiseless_selectors(numpy.stack([numpy.zeros(m, int), numpy.ones(m, int)], 1))
    got = WR.scatter(table[None], WR.assemble(None, b, m), R.transform(sel), 2 * numpy.arange(m)[None, :] + bits, m)[0]
    want = table.astype(numpy.int64)
    for q in range(Q):
        for w in range(W):
            pos = (w << m) + idx[q]                     # the layout: entry (w, i) at w 2^m + i of the flattened leaves
            want[pos >> 10, 1, pos & (N - 1)] += b[q, w]
    assert numpy.array_equal(got, (want & 0xffffffff).astype(numpy.uint32).view(numpy.int32))


def test_reference_assemble_places_columns():
    """V's coefficient 0 of column w lands at w 2^m, negacyclically"""
    rng = numpy.random.RandomState(3)
    v = rng.randint(-2**31, 2**31, size=(2, 4, 2, N)).astype(numpy.int32)
    b = rng.randint(-2**31, 2**31, size=(2, 4)).astype(numpy.int32)
    d = WR.assemble(v, b, 8)
    one = WR.assemble(v[:, 3:], b[:, 3:], 8)
    assert d.shape == (2, 1, 2, N)
    # a single column at w = 0 is (0, b) - V exactly
    want = (-(v[:, 3:].astype(numpy.int64))) & 0xffffffff
    want[:, :, 1, 0] = (want[:, :, 1, 0] + b[:, 3:]) & 0xffffffff
    assert numpy.array_equal(one.astype(numpy.int64) & 0xffffffff, want)


# ---- the Python layer on the engine double -----------------------------------------------------------------------

@pytest.fixture(scope='module')
def env():
    thr = IndexWriteFakeEngine()
    ctx = nufhe_b200.Context(rng=DeterministicRNG(20261021), thread=thr)
    sks, cks, tks, iks = [], [], [], []
    for _ in range(2):
        sk = ctx.make_secret_key()
        ck, tk, ik = ctx.make_cloud_key(sk, tree_key=True, index_key=True)
        sks.append(sk), cks.append(ck), tks.append(tk), iks.append(ik)
    vms = [ctx.make_virtual_machine(ck) for ck in cks]
    return dict(ctx=ctx, thr=thr, sks=sks, cks=cks, tks=tks, iks=iks, vms=vms)


def _read(ctx, vm, sk, ik, table, bits):
    """Every entry of the table, looked up by encrypted index and decrypted."""
    m = table.bits
    res = vm.lookup(ctx.encrypt_index(ik, numpy.arange(1 << m), m), table)
    res = [res] if table.single else res
    if table.out == 'bool':
        return numpy.stack([ctx.decrypt(sk, r) for r in res])
    return numpy.stack([ctx.decrypt_int(sk, r, bits) for r in res])


@pytest.mark.parametrize('m, W', [(3, 1), (3, 2), (11, 1)])
def test_scatter_add_counts_and_values(env, m, W):
    """plain counts into a table of zeros (repeated indexes add up), then LWE values: lookups return the sums"""
    ctx, vm, sk, ik, tk = (env[k] if k in ('ctx',) else env[k + 's'][0] for k in ('ctx', 'vm', 'sk', 'ik', 'tk'))
    rng = numpy.random.RandomState(m + W)
    zeros = numpy.zeros((W, 1 << m), int) if W > 1 else numpy.zeros(1 << m, int)
    t0 = vm.make_index_table(zeros, bits=2)
    idx = numpy.array([1, 5, 1, 2]) % (1 << m)
    t1 = vm.scatter_add(None, t0, ctx.encrypt_index(ik, idx, m), 1)
    want = numpy.zeros((W, 1 << m), int)
    for i in idx:
        want[:, i] += 1
    assert isinstance(t1, nufhe_b200.EncryptedIndexTable) and (t1.bits, t1.columns, t1.single) == (m, W, W == 1)
    assert numpy.array_equal(_read(ctx, vm, sk, ik, t1, 2), want)
    vals = rng.randint(0, 2, size=(W, 2))
    ct = [ctx.encrypt_int(sk, vals[w], 2) for w in range(W)]
    idx2 = numpy.array([3, 0]) % (1 << m)
    t2 = vm.scatter_add(tk, t1, ctx.encrypt_index(ik, idx2, m), ct if W > 1 else ct[0])
    for w in range(W):
        for q in range(2):
            want[w, idx2[q]] += vals[w, q]
    assert numpy.array_equal(_read(ctx, vm, sk, ik, t2, 2), want)
    assert t2.variance > t1.variance > 0


def test_write_overwrites(env):
    """write then lookup returns the new values and the other entries keep theirs, on int and bool tables"""
    ctx, vm, sk, ik, tk = env['ctx'], env['vms'][0], env['sks'][0], env['iks'][0], env['tks'][0]
    entries = numpy.array([3, 1, 2, 0, 1, 1, 3, 2])
    t = ctx.encrypt_table(ik, entries, bits=2)
    idx = numpy.array([6, 1])
    t2 = vm.write(tk, t, ctx.encrypt_index(ik, idx, 3), ctx.encrypt_int(sk, numpy.array([0, 2]), 2))
    want = entries.copy()
    want[idx] = [0, 2]
    assert numpy.array_equal(_read(ctx, vm, sk, ik, t2, 2)[0], want)
    t3 = vm.write(tk, t2, ctx.encrypt_index(ik, [4], 3), 3)           # plain values
    want[4] = 3
    assert numpy.array_equal(_read(ctx, vm, sk, ik, t3, 2)[0], want)
    bits = numpy.array([1, 0, 0, 1], bool)
    tb = ctx.encrypt_table(ik, bits, out='bool')
    tb2 = vm.write(tk, tb, ctx.encrypt_index(ik, [2], 2), ctx.encrypt(sk, numpy.array([True])))
    bits[2] = True
    assert numpy.array_equal(_read(ctx, vm, sk, ik, tb2, 1)[0], bits)
    # a written table pickles as any other
    assert ctx.load_encrypted_table(t3.dumps()) == t3


def test_argument_errors(env):
    ctx, thr, vm = env['ctx'], env['thr'], env['vms'][0]
    sk, ik, tk = env['sks'][0], env['iks'][0], env['tks'][0]
    t = ctx.encrypt_table(ik, numpy.arange(8) % 4, bits=2)
    idx = ctx.encrypt_index(ik, [1, 2], 3)
    x = ctx.encrypt_int(sk, numpy.array([1, 0]), 2)
    with pytest.raises(ValueError, match="out='int'"):
        vm.scatter_add(None, ctx.encrypt_table(ik, numpy.arange(8) % 2, out='bool'), idx, 1)
    with pytest.raises(TypeError, match='decompress'):
        vm.scatter_add(None, t, ctx.encrypt_index(ik, [1], 3, compressed=True), 1)
    for key in (None, ik, sk):
        with pytest.raises(TypeError, match='NuFHETreeKey'):
            vm.scatter_add(key, t, idx, x)
        with pytest.raises(TypeError, match='NuFHETreeKey'):
            vm.write(key, t, idx, x)
    with pytest.raises(TypeError):
        vm.scatter_add(None, numpy.zeros(8), idx, 1)
    with pytest.raises(ValueError, match='3-bit indices'):
        vm.scatter_add(None, t, ctx.encrypt_index(ik, [1], 4), 1)
    with pytest.raises(ValueError, match='shapes'):
        vm.scatter_add(tk, t, idx, ctx.encrypt_int(sk, numpy.array([1, 0, 1]), 2))
    with pytest.raises(ValueError, match='value arrays'):
        vm.scatter_add(tk, t, idx, [x, x])
    with pytest.raises(ValueError, match='broadcast'):
        vm.scatter_add(None, t, idx, [1, 2, 3])
    other_ctx = nufhe_b200.Context(rng=DeterministicRNG(5), thread=thr)
    other_sk = other_ctx.make_secret_key()
    _, other_tk = other_ctx.make_cloud_key(other_sk, tree_key=True)
    other_tk.params = nufhe_b200.NuFHEParameters(tlwe_mask_size=2)
    with pytest.raises(ValueError, match='other parameters'):
        vm.scatter_add(other_tk, t, idx, x)


def test_noise_rule():
    """the refusal thresholds re-derived from the margin rule: a 2-bit int table takes on the order of 100 one-query
    writes after a refresh, a bool table several hundred; 3-bit int tables have no margin to spend"""
    params = nufhe_b200.NuFHEParameters()
    assert IL.write_variance(params, 16, False) == pytest.approx(16 * (IL.cmux_variance(params)
                                                                       + IL.decomposition_variance(params)))
    assert IL.write_variance(params, 16) > IL.write_variance(params, 16, False)
    per_write = IL.write_variance(params, 16, False) + IL.rounding_variance(params)
    assert per_write == pytest.approx(3.05e-7, rel=0.02)
    fresh = lut.bootstrap_variance(params) + IL.packing_variance(params)
    for m, out, bits in ((8, 'int', 2), (16, 'int', 2), (16, 'int', 1), (16, 'bool', None), (20, 'bool', None)):
        limit = IL.max_table_variance(params, m, out, bits)
        n = IL.writes_before_refresh(params, m, out, bits)
        v = fresh
        for _ in range(n):
            v = IL.written_table_variance(params, v, m, 1)
            IL.check_table_variance(params, v, m, out, bits)
        with pytest.raises(ValueError, match='refresh_table'):
            IL.check_table_variance(params, IL.written_table_variance(params, v, m, 1), m, out, bits)
        assert v <= limit
    assert 50 <= IL.writes_before_refresh(params, 16, 'int', 2) <= 400
    assert IL.writes_before_refresh(params, 16, 'bool', None) >= 300
    assert IL.writes_before_refresh(params, 8, 'int', 3) == 0
    assert 0 < IL.writes_before_refresh(params, 16, 'int', 2, lwe_values=True)


def test_chain_until_refused(env, monkeypatch):
    """a chain of one-query scatter_adds on a table at the refresh level stops at exactly writes_before_refresh; the
    written tables record the noise rule's variances"""
    ctx, thr, vm, sk, ik = env['ctx'], env['thr'], env['vms'][0], env['sks'][0], env['iks'][0]
    params = sk.params
    m = 1
    base = ctx.encrypt_table(ik, numpy.array([1, 0]), bits=2)
    fresh = lut.bootstrap_variance(params) + IL.packing_variance(params)
    t = IL.EncryptedIndexTable(thr, params, m, 1, base.data, fresh, 'int', 2, single=True)
    n = IL.writes_before_refresh(params, m, 'int', 2)
    # skip the device work of the calls the noise rule accepts: only the count is under test here
    monkeypatch.setattr(index_write, 'scatter_passes', lambda *a, **k: None)
    idx = ctx.encrypt_index(ik, [0], m)
    count = 0
    with pytest.raises(ValueError, match='refresh_table'):
        while True:
            t = vm.scatter_add(None, t, idx, 0)
            count += 1
    assert count == n


@pytest.fixture(scope='module')
def mk_env(env):
    ctx = env['ctx']
    order = [0, 1, 0]
    machine = ctx.make_multi_key_machine([env['cks'][k] for k in order])
    return dict(env, order=order, machine=machine)


@pytest.mark.parametrize('m, W', [(2, 1), (11, 1), (3, 2)])
def test_multikey_bit_identical(mk_env, m, W):
    """mk.scatter_add and mk.write equal every tenant's own vm bit for bit (one tenant idle)"""
    ctx, machine, vms, iks, sks, tks, order = (mk_env[k] for k in ('ctx', 'machine', 'vms', 'iks', 'sks', 'tks', 'order'))
    rng = numpy.random.RandomState(m * 5 + W)
    shape = lambda e: e if W > 1 else e[0]
    tables = [ctx.encrypt_table(iks[order[t]], shape(rng.randint(0, 2, size=(W, 1 << m))), bits=2) for t in range(3)]
    idx = [ctx.encrypt_index(iks[order[0]], rng.randint(0, 1 << m, size=2), m), None,
           ctx.encrypt_index(iks[order[2]], rng.randint(0, 1 << m, size=(1,)), m)]
    vals = [None] * 3
    for t in (0, 2):
        cols = [ctx.encrypt_int(sks[order[t]], rng.randint(0, 2, size=idx[t].shape), 2) for _ in range(W)]
        vals[t] = cols if W > 1 else cols[0]
    keys = [tks[order[t]] for t in range(3)]
    for op in ('scatter_add', 'write'):
        out = getattr(machine, op)(keys, tables, idx, vals)
        assert out[1] is None
        for t in (0, 2):
            want = getattr(vms[order[t]], op)(keys[t], tables[t], idx[t], vals[t])
            assert out[t] == want, (op, t)
    counts = machine.scatter_add([None] * 3, tables, idx, [1, None, 2])
    for t in (0, 2):
        assert counts[t] == vms[order[t]].scatter_add(None, tables[t], idx[t], [1, None, 2][t])
    with pytest.raises(ValueError, match='tenant 2'):
        machine.scatter_add([None] * 3, tables, idx[:2] + [ctx.encrypt_index(iks[0], [1], m + 1)], [1, None, 1])
