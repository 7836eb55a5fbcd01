"""Encrypted tables on the GPU (DESIGN.md section 20): client-encrypted and server-packed tables read by vm.lookup, bit
for bit against the oracle-composed reference (tests/index_ref.py) and the oracle packing (tests/pack_ref.py); the
indirect index kernels against the existing ones; mk.lookup with one table per tenant against each tenant's own
vm.lookup, also on compressed keys in rounds; and the output noise against the section 20 estimates."""
import numpy
import pytest
import torch

import index_ref as R
import pack_ref

pytestmark = pytest.mark.gpu

N = 1024


def _rand_i32(rng, shape):
    return rng.randint(-2**31, 2**31, size=shape, dtype=numpy.int64).astype(numpy.int32)


@pytest.fixture(scope='module')
def api():
    import nufhe_b200 as nufhe
    ctx = nufhe.Context(rng=nufhe.DeterministicRNG(20261020))
    sk = ctx.make_secret_key()
    ck, tk, ik, cpk = ctx.make_cloud_key(sk, tree_key=True, index_key=True, compact_public_key=True)
    vm = ctx.make_virtual_machine(ck)
    return dict(nufhe=nufhe, ctx=ctx, sk=sk, ck=ck, tk=tk, ik=ik, cpk=cpk, vm=vm)


def _same(x, y):
    return (tuple(x.shape) == tuple(y.shape) and torch.equal(x.a, y.a) and torch.equal(x.b, y.b)
            and torch.equal(x.current_variances, y.current_variances))


@pytest.mark.parametrize('m, W', [(4, 8), (10, 1), (12, 2), (16, 1)])
def test_compact_key_tables(api, m, W):
    """a table encrypted with the compact public key, 4096 random indices: the results decrypt to table[idx]"""
    ctx, sk, ik, cpk, vm = (api[k] for k in ('ctx', 'sk', 'ik', 'cpk', 'vm'))
    rng = numpy.random.RandomState(m)
    tab = rng.randint(0, 4, size=(W, 1 << m))
    values = rng.randint(0, 1 << m, size=4096)
    values[:2] = 0, (1 << m) - 1
    t = ctx.encrypt_table(cpk, tab if W > 1 else tab[0], bits=2)
    res = vm.lookup(ctx.encrypt_index(ik, values, m), ctx.load_encrypted_table(t.dumps()))
    res = res if W > 1 else [res]
    for w in range(W):
        assert numpy.array_equal(ctx.decrypt_int(sk, res[w], 2), tab[w][values]), w


@pytest.mark.parametrize('m, W, Q', [(4, 8, 3), (11, 1, 3), (11, 2, 5)])
def test_small_batch_matches_oracle(api, m, W, Q):
    """the lookup before the key switch of a compact-key table, random selector rows, bit for bit against the
    reference composed from the oracle's external product"""
    nufhe, ctx, cpk = api['nufhe'], api['ctx'], api['cpk']
    from nufhe_b200 import index_lookup as IL
    rng = numpy.random.RandomState(m * 7 + Q)
    t = ctx.encrypt_table(cpk, rng.randint(0, 8, size=(W, 1 << m)), bits=3)
    rows = _rand_i32(rng, (Q, m, 2, 2, 2, N))
    index = IL.EncryptedIndexArray(cpk.params, m, ctx.thread.to_device(rows), 0.0)
    a, b = IL.lookup_extracted(ctx.thread, index, t)
    wa, wb = R.lookup(t.nodes.cpu().numpy(), R.transform(rows), numpy.arange(Q * m).reshape(Q, m), m, W)
    assert numpy.array_equal(a.cpu().numpy(), wa) and numpy.array_equal(b.cpu().numpy(), wb)


def test_zero_mask_table_equals_plaintext_table(api):
    """zero masks and bodies equal to the plaintext encoding: vm.lookup gives exactly the IndexTable's results"""
    ctx, ik, vm = api['ctx'], api['ik'], api['vm']
    from nufhe_b200 import index_lookup as IL
    rng = numpy.random.RandomState(12)
    m, W = 12, 2
    plain = vm.make_index_table(rng.randint(0, 4, size=(W, 1 << m)), bits=2)
    data = numpy.zeros((IL.table_polys_count(m, W), 2, N), numpy.uint16)
    data[:, 1] = (plain.polys.cpu().numpy()[:, 1].view(numpy.uint32) >> 16).astype(numpy.uint16)
    enc = IL.EncryptedIndexTable(ctx.thread, plain.params, m, W, ctx.thread.to_device(data), 0.0, 'int', 2)
    idx = ctx.encrypt_index(ik, rng.randint(0, 1 << m, size=257), m)
    for got, want in zip(vm.lookup(idx, enc), vm.lookup(idx, plain)):
        assert _same(got, want)


def _tree_key_polys(tk):
    from chacha_ref import seeded_uniform
    k = tk.params.tgsw_params.tlwe_params.mask_size
    return pack_ref.key_polys(seeded_uniform(tk.seed, 5, (500, 2, k, N)), tk.body.cpu().numpy())


def test_server_packed_table(api):
    """a table packed from gate_nand outputs with the tree key: the nodes are bit-identical to the oracle packing with
    the tree key's masks and bodies; lookups decrypt to the outputs and feed gate_nand; a table packed from LUT outputs
    feeds vm.lut"""
    ctx, sk, ik, tk, vm = (api[k] for k in ('ctx', 'sk', 'ik', 'tk', 'vm'))
    rng = numpy.random.RandomState(5)
    m = 10
    p, q = rng.randint(0, 2, size=(2, 1 << m)).astype(bool)
    col = vm.gate_nand(ctx.encrypt(sk, p), ctx.encrypt(sk, q))
    t = vm.make_encrypted_table(tk, col, out='bool')
    want = pack_ref.pack(col.a.cpu().numpy(), col.b.cpu().numpy(), _tree_key_polys(tk))
    assert (t.data.cpu().numpy() == want).all()
    values = rng.randint(0, 1 << m, size=4096)
    r = vm.lookup(ctx.encrypt_index(ik, values, m), t)
    truth = ~(p & q)
    assert numpy.array_equal(ctx.decrypt(sk, r), truth[values])
    assert numpy.array_equal(ctx.decrypt(sk, vm.gate_nand(r, r)), ~truth[values])
    # LUT outputs: f(x) packed with 2-bit entries, read back and fed to g
    x = rng.randint(0, 4, size=(2, 1 << 12))
    f = vm.make_lut([1, 2, 3, 0], 2)
    cols = vm.lut(f, ctx.encrypt_int(sk, x, 2))
    t2 = vm.make_encrypted_table(tk, cols, out='int', bits=2)
    assert (t2.bits, t2.columns) == (12, 2)
    values = rng.randint(0, 1 << 12, size=4096)
    r0, r1 = vm.lookup(ctx.encrypt_index(ik, values, 12), t2)
    g = vm.make_lut([3, 2, 1, 0], 2)
    fx = (x + 1) % 4
    assert numpy.array_equal(ctx.decrypt_int(sk, r1, 2), fx[1][values])
    assert numpy.array_equal(ctx.decrypt_int(sk, vm.lut(g, r0), 2), 3 - fx[0][values])


@pytest.mark.parametrize('Q', [1, 2, 3, 257, 4096])
def test_indirect_kernels_match_direct(api, Q):
    """the indirect levels with every query on one table equal the existing kernels on that shared table; with three
    tables (neighbouring queries, so the two slots of a CTA, on different tables, and an odd Q replaying the last slot)
    they equal the existing kernels on per-query copies"""
    eng = api['ctx'].thread
    rng = numpy.random.RandomState(Q)
    for m, W in ((11, 1), (8, 4), (10, 2)):
        P = W << max(m - 10, 0) if m >= 10 else 1
        tables = eng.to_device(_rand_i32(rng, (3, P, 2, N)))
        sel = eng.to_device(_rand_i32(rng, (min(Q, 8), m, 2, 2, 2, N)))[torch.arange(Q, device=eng.device) % min(Q, 8)]
        spec = eng.index_prepare(sel).reshape(Q, m, -1)
        for ids in (numpy.zeros(Q, numpy.uint32), (numpy.arange(Q) % 3).astype(numpy.uint32)):
            one = tables[0] if not ids.any() else tables[torch.from_numpy(ids.astype(numpy.int64)).to(eng.device)]
            if m > 10:
                got = eng.index_cmux_level_indirect(tables, ids, spec, 10, Q)
                assert torch.equal(got, eng.index_cmux_level(one, spec, 10, Q)), (m, ids[:3])
            else:
                ga, gb = eng.index_rotate_extract_indirect(tables, ids, spec, m, W, Q)
                wa, wb = eng.index_rotate_extract(one, spec, m, W, Q)
                assert torch.equal(ga, wa) and torch.equal(gb, wb), (m, ids[:3])
    with pytest.raises(Exception):
        eng.index_rotate_extract_indirect(tables, numpy.full(Q, 3, numpy.uint32), spec, 10, 2, Q)


@pytest.fixture(scope='module')
def tenants():
    import nufhe_b200 as nufhe
    ctx = nufhe.Context(rng=nufhe.DeterministicRNG(20261021))
    keys = []
    for _ in range(3):
        sk = ctx.make_secret_key()
        cck, ik, cpk = ctx.make_cloud_key(sk, compressed=True, index_key=True, compact_public_key=True)
        keys.append((sk, cck, ik, cpk))
    vms = [ctx.make_virtual_machine(k[1].decompress(ctx.thread)) for k in keys]
    return ctx, keys, vms


@pytest.mark.parametrize('m', [8, 12])
def test_multikey_per_tenant_tables(tenants, m):
    """3 tenants with their own tables, one idle: each tenant's results equal its own vm.lookup bit for bit, on
    resident keys and on compressed keys with resident_tenants=2 (rounds); a shared IndexTable keeps today's results"""
    ctx, keys, vms = tenants
    rng = numpy.random.RandomState(m)
    W = 2
    tabs = [rng.randint(0, 4, size=(W, 1 << m)) for _ in range(4)]
    tables = [ctx.encrypt_table(keys[t][3] if t != 1 else keys[t][2], tabs[t], bits=2) for t in range(3)] + [None]
    order = [0, 1, 2, 0]
    vals = [rng.randint(0, 1 << m, size=s) for s in (300, 1, 257)] + [None]
    idx = [None if v is None else ctx.encrypt_index(keys[order[t]][2], v, m) for t, v in enumerate(vals)]
    resident = ctx.make_multi_key_machine([vm.cloud_key for vm in (vms[0], vms[1], vms[2], vms[0])])
    pooled = ctx.make_multi_key_machine([keys[k][1] for k in order], resident_tenants=2)
    plain = vms[0].make_index_table(tabs[3], bits=2)
    for machine in (resident, pooled):
        out = machine.lookup(idx, tables)
        assert out[3] is None
        for t in range(3):
            want = vms[order[t]].lookup(idx[t], tables[t])
            assert all(_same(g, w) for g, w in zip(out[t], want)), t
            for w in range(W):
                assert numpy.array_equal(ctx.decrypt_int(keys[order[t]][0], out[t][w], 2), tabs[t][w][vals[t]])
        shared = machine.lookup(idx, plain)
        for t in range(3):
            assert all(_same(g, w) for g, w in zip(shared[t], vms[order[t]].lookup(idx[t], plain))), t


@pytest.mark.parametrize('kind, m, W', [('compact', 10, 16), ('compact', 16, 4), ('packed', 10, 16), ('packed', 16, 1)])
def test_output_noise(api, kind, m, W):
    """4096 queries, phases before the key switch: the variance of the error against the table lies within 0.5 to 2
    times the estimate (leaf variance + extracted_variance) and no error exceeds 7 sigma.  The error the lookup itself
    adds (against the table's encoding for compact leaves, against the packed inputs' own phases for packed leaves, whose
    bootstrap outputs carry their own mean shift) has a mean below a tenth of its standard deviation; for packed leaves
    its variance lies within 0.5 to 2 times packing_variance + extracted_variance"""
    nufhe, ctx, sk, ik, cpk, tk, vm = (api[k] for k in ('nufhe', 'ctx', 'sk', 'ik', 'cpk', 'tk', 'vm'))
    from nufhe_b200 import index_lookup as IL
    params = nufhe.NuFHEParameters()
    rng = numpy.random.RandomState(m * 3 + W)
    tab = rng.randint(0, 4, size=(W, 1 << m))
    want = None
    if kind == 'compact':
        t = ctx.encrypt_table(cpk, tab, bits=2)
    else:
        cols = vm.lut(vm.make_lut([0, 1, 2, 3], 2), ctx.encrypt_int(sk, tab, 2))
        t = vm.make_encrypted_table(tk, cols, bits=2)
        s = sk.lwe_key.key.to(cols.a.device)
        n = cols.a.shape[-1]
        want = ctx.thread.lwe_dot(cols.a.reshape(-1, n), s, add1=cols.b.reshape(-1), sign=-1).cpu().numpy()
        want = want.astype(numpy.int64).reshape(W, -1)
    values = rng.randint(0, 1 << m, size=4096)
    a, b = IL.lookup_extracted(ctx.thread, ctx.encrypt_index(ik, values, m), t)
    key = ik.key.reshape(-1).to(a.device)
    phase = ctx.thread.lwe_dot(a.reshape(-1, N), key, add1=b.reshape(-1), sign=-1).cpu().numpy().reshape(W, -1)
    centred = lambda x: ((x + 2**31) % 2**32 - 2**31) / 2**32
    err = centred(phase.astype(numpy.int64) - (tab[:, values].astype(numpy.int64) << 29))
    var = float((err**2).mean())
    est = t.variance + IL.extracted_variance(params, m)
    own = err if want is None else centred(phase.astype(numpy.int64) - want[:, values])
    own_est = IL.extracted_variance(params, m) + (t.variance if want is None else IL.packing_variance(params))
    own_var = float((own**2).mean())
    print('%s m = %d: variance %.3g, estimate %.3g (ratio %.2f), max |err| %.3g, mean %.3g; the lookup alone %.3g, '
          'estimate %.3g (ratio %.2f), mean %.3g' % (kind, m, var, est, var / est, abs(err).max(), err.mean(), own_var,
                                                     own_est, own_var / own_est, own.mean()))
    assert 0.5 * est <= var <= 2 * est
    assert abs(err).max() < 7 * est**0.5
    assert 0.5 * own_est <= own_var <= 2 * own_est
    assert abs(own.mean()) < 0.1 * own_est**0.5
