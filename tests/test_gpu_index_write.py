"""Oblivious writes on the GPU (DESIGN.md section 21): the assembly, rotation and demultiplexer kernels bit for bit
against the oracle-composed reference (tests/write_ref.py) at several batch sizes and bit counts, a collision of every
query on one index, scatter_add / write / refresh_table end to end through lookups, mk.scatter_add / mk.write against
each tenant's own vm, and the measured per-write noise against the estimate."""
import numpy
import pytest
import torch

import index_ref as R
import write_ref as WR

pytestmark = pytest.mark.gpu

N = 1024


def _rand_i32(rng, shape):
    return rng.randint(-2**31, 2**31, size=shape, dtype=numpy.int64).astype(numpy.int32)


@pytest.fixture(scope='module')
def api():
    import nufhe_b200 as nufhe
    ctx = nufhe.Context(rng=nufhe.DeterministicRNG(20261021))
    sk = ctx.make_secret_key()
    ck, tk, ik = ctx.make_cloud_key(sk, tree_key=True, index_key=True)
    vm = ctx.make_virtual_machine(ck)
    return dict(nufhe=nufhe, ctx=ctx, sk=sk, ck=ck, tk=tk, ik=ik, vm=vm)


def _kernels_vs_reference(api, m, W, Q, idx=None, lwe=True):
    from nufhe_b200 import index_write
    from nufhe_b200.batch_keys import OneKey
    ctx, ik, tk, sk = api['ctx'], api['ik'], api['tk'], api['sk']
    thr = ctx.thread
    params = sk.params
    rng = numpy.random.RandomState(m * 1000 + Q)
    if idx is None:
        idx = rng.randint(0, 1 << m, size=Q)
    sels = ctx.encrypt_index(ik, idx, m).samples.reshape(Q, m, 2, 2, 2, N)
    P = (W << (m - 10)) if m >= 10 else 1
    nodes = _rand_i32(rng, (P, 2, N))
    n = params.in_out_params.size
    a = thr.to_device(_rand_i32(rng, (Q, W, n))) if lwe else None
    b = thr.to_device(_rand_i32(rng, (Q, W)))
    acc = thr.to_device(nodes)[None].contiguous()
    index_write.scatter_passes(thr, params, OneKey(thr, tree_key=tk), m, W, [sels], a, b, acc)
    v = thr.tree_keyswitch(a.reshape(Q * W, n), tk.planes(thr), 1).reshape(Q, W, 2, N) if lwe else None
    delta = WR.assemble(None if v is None else v.cpu().numpy(), b.cpu().numpy(), m)
    assert numpy.array_equal(thr.index_write_assemble(v, b, m).cpu().numpy(), delta)
    rows = numpy.arange(Q)[:, None] * m + numpy.arange(m)[None, :]
    want = WR.scatter(nodes[None], delta, R.transform(sels.cpu().numpy()), rows, m)
    assert numpy.array_equal(acc.cpu().numpy(), want)


@pytest.mark.parametrize('Q', [1, 2, 3, 64, 257, 4096])
def test_batch_sizes_match_oracle(api, Q):
    _kernels_vs_reference(api, 11, 1, Q)


@pytest.mark.parametrize('m, W, Q', [(1, 3, 5), (8, 4, 5), (10, 2, 3), (16, 1, 3), (20, 1, 2)])
def test_bit_counts_match_oracle(api, m, W, Q):
    _kernels_vs_reference(api, m, W, Q, lwe=m != 8)


def test_collision_matches_oracle(api):
    """every query on one index: the atomics add them all, in whatever order"""
    _kernels_vs_reference(api, 11, 1, 300, idx=numpy.full(300, 1234))
    _kernels_vs_reference(api, 6, 2, 300, idx=numpy.full(300, 17))


def _read(api, table, bits):
    ctx, vm, sk, ik = api['ctx'], api['vm'], api['sk'], api['ik']
    m = table.bits
    res = vm.lookup(ctx.encrypt_index(ik, numpy.arange(1 << m), m), table)
    res = [res] if table.single else res
    if table.out == 'bool':
        return numpy.stack([ctx.decrypt(sk, r) for r in res])
    return numpy.stack([ctx.decrypt_int(sk, r, bits) for r in res])


@pytest.mark.parametrize('m', [4, 12])
def test_scatter_add_end_to_end(api, m):
    """plain counts (a histogram of 500 votes) then LWE values computed by the server, then lookups"""
    ctx, vm, sk, ik, tk = (api[k] for k in ('ctx', 'vm', 'sk', 'ik', 'tk'))
    rng = numpy.random.RandomState(m)
    votes = rng.randint(0, 1 << m, size=500) % 8 if m > 4 else rng.randint(0, 16, size=500)
    t = vm.scatter_add(None, vm.make_index_table(numpy.zeros(1 << m, int), bits=2), ctx.encrypt_index(ik, votes[:3], m), 1)
    want = numpy.bincount(votes[:3], minlength=1 << m)
    assert numpy.array_equal(_read(api, t, 2)[0], want % 4)
    x = ctx.encrypt_int(sk, numpy.array([1, 2]), 2)
    y = vm.lut(vm.make_lut(numpy.array([0, 1, 2, 3]), 2), x)          # computed on the server
    idx = numpy.array([5, 7]) % (1 << m)
    t2 = vm.scatter_add(api['tk'], t, ctx.encrypt_index(ik, idx, m), y)
    want[idx] += [1, 2]
    assert numpy.array_equal(_read(api, t2, 2)[0], want % 4)


def test_write_end_to_end_and_refresh(api):
    """write then lookup returns the new values and the others keep theirs; a chain of writes until ValueError, then
    refresh_table, then more writes"""
    ctx, vm, sk, ik, tk = (api[k] for k in ('ctx', 'vm', 'sk', 'ik', 'tk'))
    from nufhe_b200 import index_lookup as IL
    m = 6
    rng = numpy.random.RandomState(1)
    entries = rng.randint(0, 4, size=(2, 1 << m))
    t = ctx.encrypt_table(ik, entries, bits=2)
    idx = numpy.array([3, 40, 63])
    new = rng.randint(0, 4, size=(2, 3))
    t = vm.write(tk, t, ctx.encrypt_index(ik, idx, m), [ctx.encrypt_int(sk, new[w], 2) for w in range(2)])
    entries[:, idx] = new
    assert numpy.array_equal(_read(api, t, 2), entries)
    bits = rng.randint(0, 2, size=1 << m).astype(bool)
    tb = vm.write(tk, ctx.encrypt_table(ik, bits, out='bool'), ctx.encrypt_index(ik, [9], m),
                  ctx.encrypt(sk, numpy.array([not bits[9]])))
    bits[9] = not bits[9]
    assert numpy.array_equal(_read(api, tb, 1)[0], bits)
    count = 0
    with pytest.raises(ValueError, match='refresh_table'):
        while True:
            i = count % (1 << m)
            t = vm.write(tk, t, ctx.encrypt_index(ik, [i], m), entries[:, i][:, None].tolist())
            count += 1
    assert count >= 1
    assert numpy.array_equal(_read(api, t, 2), entries)
    r = vm.refresh_table(tk, t)
    assert r.variance == pytest.approx(IL.lut.bootstrap_variance(sk.params) + IL.packing_variance(sk.params))
    assert numpy.array_equal(_read(api, r, 2), entries)
    r = vm.write(tk, r, ctx.encrypt_index(ik, [0], m), [[1], [2]])
    entries[:, 0] = [1, 2]
    assert numpy.array_equal(_read(api, r, 2), entries)
    rb = vm.refresh_table(tk, tb)
    assert numpy.array_equal(_read(api, rb, 1)[0], bits)


def test_multikey_bit_identical(api):
    nufhe, ctx = api['nufhe'], api['ctx']
    sks, cks, tks, iks = [], [], [], []
    for _ in range(2):
        sk = ctx.make_secret_key()
        ck, tk, ik = ctx.make_cloud_key(sk, tree_key=True, index_key=True)
        sks.append(sk), cks.append(ck), tks.append(tk), iks.append(ik)
    machine = ctx.make_multi_key_machine(cks)
    vms = [ctx.make_virtual_machine(ck) for ck in cks]
    rng = numpy.random.RandomState(2)
    for m in (5, 11):
        tables = [ctx.encrypt_table(iks[t], rng.randint(0, 4, size=1 << m), bits=2) for t in range(2)]
        idx = [ctx.encrypt_index(iks[t], rng.randint(0, 1 << m, size=3 + 60 * t), m) for t in range(2)]
        vals = [ctx.encrypt_int(sks[t], rng.randint(0, 2, size=idx[t].shape), 2) for t in range(2)]
        for op in ('scatter_add', 'write'):
            out = getattr(machine, op)(tks, tables, idx, vals)
            for t in range(2):
                assert out[t] == getattr(vms[t], op)(tks[t], tables[t], idx[t], vals[t]), (m, op, t)


@pytest.mark.parametrize('m', [8, 16])
def test_write_noise(api, m):
    """the noise one scatter_add of Q server LWE values adds to the entries it does not write, from phases decrypted
    with S, against Q write_variance + rounding_variance (the tree-key-switched deltas have uniform masks, so the
    digits the selectors multiply are uniform, as the estimate assumes).  Up to m = 10 every entry takes all m products
    and the estimate is met; above, an entry outside the written leaf takes only the demultiplexer levels below the
    one where its path leaves the written leaf's, and the estimate is an upper bound"""
    from nufhe_b200 import index_lookup as IL
    from oracle import oracle as O
    ctx, vm, ik, sk, tk = api['ctx'], api['vm'], api['ik'], api['sk'], api['tk']
    Q = 64
    rng = numpy.random.RandomState(m)
    idx = rng.randint(0, 1 << m, size=Q)
    t = vm.scatter_add(tk, vm.make_index_table(numpy.zeros(1 << m, int), bits=2), ctx.encrypt_index(ik, idx, m),
                       ctx.encrypt_int(sk, numpy.zeros(Q, int), 2))
    nodes = t.nodes.cpu().numpy()
    S = ik.key.cpu().numpy()[0]
    prod = O.poly_mul_i32(S, numpy.ascontiguousarray(nodes[:, 0])).reshape(-1, N)
    ph = ((nodes[:, 1].astype(numpy.int64) - prod.astype(numpy.int64)) & 0xffffffff).reshape(-1)[:1 << m]
    ph = numpy.delete(numpy.where(ph >= 2**31, ph - 2**32, ph) / 2.0**32, numpy.unique(idx))
    measured = float(numpy.mean(ph**2))
    est = Q * IL.write_variance(sk.params, m) + IL.rounding_variance(sk.params)
    print('m = %d: measured %.3e, estimate %.3e, ratio %.3f' % (m, measured, est, measured / est))
    if m <= 10:
        assert 0.8 < measured / est < 1.2
    else:
        assert 0 < measured / est < 1.1
    assert t.variance >= est
