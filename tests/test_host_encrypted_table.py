"""CPU tests of encrypted tables (nufhe_b200/index_lookup.py: EncryptedIndexTable, DESIGN.md section 20): the
oracle-composed lookup (tests/index_ref.py) on GLWE leaves with non-zero masks, the layout of client-encrypted tables,
pickles, argument errors and the noise functions, server-packed tables, and per-tenant tables on the multi-key machine,
all on the oracle-backed engine double."""
import numpy
import pytest
import torch

import nufhe_b200
from nufhe_b200 import index_lookup as IL
from nufhe_b200 import lut, packing
from nufhe_b200.gates import MU
from nufhe_b200.random_numbers import DeterministicRNG
from encrypted_table_fake import EncryptedTableFakeEngine
from oracle import oracle as O
import index_ref as R

N = 1024


# ---- the reference -----------------------------------------------------------------------------------------------

def _phase(nodes, S):
    """body - S mask of GLWE samples (..., 2, N) int32, int64 mod 2^32."""
    c = numpy.ascontiguousarray(nodes).reshape(-1, 2, N)
    prod = O.poly_mul_i32(S, numpy.ascontiguousarray(c[:, 0])).reshape(-1, N)
    return ((c[:, 1].astype(numpy.int64) - prod.astype(numpy.int64)) & 0xffffffff).reshape(nodes.shape[:-2] + (N,))


@pytest.mark.parametrize('m, W', [(3, 2), (10, 1), (11, 2)])
def test_reference_reads_glwe_leaves(m, W):
    """random GLWE leaves (non-zero masks, every word a multiple of 2^12 so that the rounded decomposition is exact)
    and trivial selectors b H: the extracted sample of every query decrypts under S to the leaf's phase at the entry's
    coefficient, exactly"""
    rng = numpy.random.RandomState(m + W)
    P = IL.table_polys_count(m, W)
    leaves = (rng.randint(0, 2**20, size=(P, 2, N)).astype(numpy.int64) << 12).astype(numpy.uint32).view(numpy.int32)
    S = rng.randint(0, 2, size=N).astype(numpy.int32)
    idx = numpy.concatenate([[0, (1 << m) - 1], rng.randint(0, 1 << m, size=6)])
    bits = (idx[:, None] >> numpy.arange(m)) & 1
    sel = R.noiseless_selectors(numpy.stack([numpy.zeros(m, int), numpy.ones(m, int)], 1))
    a, b = R.lookup(leaves, R.transform(sel), 2 * numpy.arange(m)[None, :] + bits, m, W)
    leaf_phase = _phase(leaves, S).reshape(-1)                  # entry (w, i) of the layout at w 2^m + i
    for w in range(W):
        got = (b[w].astype(numpy.int64) - (a[w].astype(numpy.int64) * S[None, :]).sum(1)) & 0xffffffff
        assert numpy.array_equal(got, leaf_phase[(w << m) + idx]), w


# ---- the Python layer on the engine double -----------------------------------------------------------------------

@pytest.fixture(scope='module')
def env():
    thr = EncryptedTableFakeEngine()
    ctx = nufhe_b200.Context(rng=DeterministicRNG(20261019), thread=thr)
    sks, cks, tks, iks, cpks = [], [], [], [], []
    for _ in range(2):
        sk = ctx.make_secret_key()
        ck, tk, ik, cpk = ctx.make_cloud_key(sk, tree_key=True, index_key=True, compact_public_key=True)
        for lst, v in zip((sks, cks, tks, iks, cpks), (sk, ck, tk, ik, cpk)):
            lst.append(v)
    vms = [ctx.make_virtual_machine(ck) for ck in cks]
    return dict(ctx=ctx, thr=thr, sks=sks, cks=cks, tks=tks, iks=iks, cpks=cpks, vms=vms)


def _same(x, y):
    return (tuple(x.shape) == tuple(y.shape) and (x.a == y.a).all() and (x.b == y.b).all()
            and (x.current_variances == y.current_variances).all())


def _centred(x):
    x = numpy.asarray(x, numpy.int64) & 0xffffffff
    return numpy.where(x >= 2**31, x - 2**32, x)


@pytest.mark.parametrize('m, W', [(1, 1), (4, 3), (9, 2), (10, 1), (10, 2), (11, 3), (13, 1)])
def test_layout_round_trip(env, m, W):
    """a table encrypted with the index secret key decrypts under S to IndexTable's plaintext layout (0 in unused
    coefficients), within the fresh noise and the 16-bit rounding; nodes are data << 16"""
    ctx, ik = env['ctx'], env['iks'][0]
    rng = numpy.random.RandomState(m * 10 + W)
    entries = rng.randint(0, 8, size=(W, 1 << m))
    t = ctx.encrypt_table(ik, entries if W > 1 else entries[0], bits=3)
    assert isinstance(t, nufhe_b200.EncryptedIndexTable) and (t.bits, t.columns, t.single) == (m, W, W == 1)
    P = IL.table_polys_count(m, W)
    assert tuple(t.data.shape) == (P, 2, N) and t.data.dtype == torch.uint16
    data = t.data.view(torch.int16).numpy().astype(numpy.int64) & 0xffff
    assert numpy.array_equal(t.nodes.numpy().astype(numpy.int64) & 0xffffffff, data << 16)
    want = R.table_polys(lut.encode_int(entries, 3), m)[:, 1]
    err = _centred(_phase(t.nodes.numpy(), ik.key.numpy()[0]) - want)
    assert numpy.abs(err).max() < 2**24
    assert t.variance == pytest.approx(IL.rounding_variance(ik.params), rel=1e-6)


@pytest.mark.parametrize('m, W', [(4, 3), (11, 1)])
def test_compact_key_tables(env, m, W):
    """a compact public key encrypts the flattened layout with compact_encrypt's draws"""
    ctx, thr, cpk, ik = env['ctx'], env['thr'], env['cpks'][0], env['iks'][0]
    rng = numpy.random.RandomState(m)
    entries = rng.randint(0, 2, size=(W, 1 << m))
    state = ctx.rng.rng.get_state()
    t = ctx.encrypt_table(cpk, entries, out='bool')
    ctx.rng.rng.set_state(state)
    plain = numpy.where(entries != 0, int(MU), -int(MU)).astype(numpy.int32)
    want = R.table_polys(plain, m)[:, 1]
    same = nufhe_b200.compact_encrypt(thr, ctx.rng, cpk, thr.to_device(want))
    assert numpy.array_equal(t.data.numpy(), same.data.numpy())
    err = _centred(_phase(t.nodes.numpy(), ik.key.numpy()[0]) - want)
    assert numpy.abs(err).max() < 2**24
    fresh, mr, br, _ = nufhe_b200.compact.noise_terms(cpk.params)
    assert t.variance == fresh + mr + br and t.out == 'bool' and not t.single


def test_zero_mask_table_equals_plaintext_table(env):
    """an encrypted table with zero masks and bodies equal to the plaintext encoding gives exactly IndexTable's
    result; its leaf variance 0 leaves the recorded variance as IndexTable's"""
    ctx, thr, vm, ik, sk = env['ctx'], env['thr'], env['vms'][0], env['iks'][0], env['sks'][0]
    for m, W in ((3, 2), (11, 1)):
        rng = numpy.random.RandomState(m)
        entries = rng.randint(0, 4, size=(W, 1 << m))
        plain = vm.make_index_table(entries, bits=2)
        data = numpy.zeros((IL.table_polys_count(m, W), 2, N), numpy.uint16)
        data[:, 1] = (plain.polys.numpy()[:, 1].view(numpy.uint32) >> 16).astype(numpy.uint16)
        enc = IL.EncryptedIndexTable(thr, sk.params, m, W, thr.to_device(data), 0.0, 'int', 2, single=False)
        assert torch.equal(enc.nodes, plain.polys)
        idx = ctx.encrypt_index(ik, rng.randint(0, 1 << m, size=3), m)
        for got, want in zip(vm.lookup(idx, enc), vm.lookup(idx, plain)):
            assert _same(got, want)


def test_lookup_into_encrypted_table(env):
    """client-encrypted leaves: results decrypt to table[idx] and record leaf + lookup variance"""
    ctx, vm, ik, sk, cpk = env['ctx'], env['vms'][0], env['iks'][0], env['sks'][0], env['cpks'][0]
    entries = numpy.arange(32).reshape(2, 16) % 8
    for key in (ik, cpk):
        t = ctx.encrypt_table(key, entries, bits=3)
        vals = numpy.array([[0, 15], [7, 9]])
        res = vm.lookup(ctx.encrypt_index(ik, vals, 4), t)
        for w in range(2):
            assert (ctx.decrypt_int(sk, res[w], 3) == entries[w][vals]).all()
            assert (res[w].current_variances.numpy() == numpy.float32(t.variance + IL.output_variance(sk.params, 4))).all()


def test_pickles_round_trip(env):
    ctx, ik = env['ctx'], env['iks'][0]
    t = ctx.encrypt_table(ik, numpy.arange(8) % 2, out='bool')
    s = t.dumps()
    assert b'nufhe_b200.EncryptedIndexTable/1' in s
    u = ctx.load_encrypted_table(s)
    assert u == t and torch.equal(u.nodes, t.nodes) and u.single
    t2 = ctx.encrypt_table(ik, numpy.arange(2048).reshape(2, 1024) % 4, bits=2)
    assert ctx.load_encrypted_table(t2.dumps()) == t2
    assert len(t2.dumps()) - 2 * 2 * N * 2 * 2 < 1024           # 4 bytes per entry and a small header
    for wrong in (ik.dumps(), ctx.encrypt_index(ik, [1], 3).dumps(), b'not a pickle', s[:-100]):
        with pytest.raises(ValueError):
            ctx.load_encrypted_table(wrong)


def test_argument_errors(env):
    ctx, thr, vm = env['ctx'], env['thr'], env['vms'][0]
    ik, sk, ck, tk, cpk = (env[k][0] for k in ('iks', 'sks', 'cks', 'tks', 'cpks'))
    for key in (sk, ck, tk, None):
        with pytest.raises(TypeError):
            ctx.encrypt_table(key, numpy.arange(8) % 2, out='bool')
    # the same caps and messages as IndexTable
    for table, kw in ((numpy.zeros(3), {'out': 'bool'}), (numpy.zeros((5, 256)), {'out': 'bool'}),
                      (numpy.zeros(1 << 21), {'out': 'bool'}), (numpy.zeros(8), {'out': 'float'}),
                      (numpy.zeros(8), {'out': 'int'}), (numpy.full(8, 4), {'out': 'int', 'bits': 2}),
                      (numpy.zeros(8), {'out': 'int', 'bits': 4})):
        with pytest.raises(ValueError) as plain:
            IL.IndexTable(thr, sk.params, table, **kw)
        for key in (ik, cpk):
            with pytest.raises(ValueError) as enc:
                ctx.encrypt_table(key, table, **kw)
            assert str(enc.value) == str(plain.value)
    t = ctx.encrypt_table(ik, numpy.arange(8) % 4, bits=2)
    with pytest.raises(ValueError, match='3-bit indices'):
        vm.lookup(ctx.encrypt_index(ik, [1], 4), t)
    with pytest.raises(ValueError):
        IL.EncryptedIndexTable(thr, sk.params, 3, 1, t.data[:, :1], 0.0, 'int', 2)
    # server-packed tables
    x = ctx.encrypt(sk, numpy.zeros(8, bool))
    with pytest.raises(TypeError):
        vm.make_encrypted_table(thr, x, out='bool')
    with pytest.raises(TypeError):
        vm.make_encrypted_table(ik, x, out='bool')
    with pytest.raises(ValueError, match='2\\^m entries'):
        vm.make_encrypted_table(tk, ctx.encrypt(sk, numpy.zeros(6, bool)), out='bool')
    with pytest.raises(ValueError, match='one shape'):
        vm.make_encrypted_table(tk, [x, ctx.encrypt(sk, numpy.zeros(4, bool))], out='bool')
    with pytest.raises(ValueError):
        vm.make_encrypted_table(tk, x, out='int', bits=4)
    with pytest.raises(ValueError):
        vm.make_encrypted_table(tk, x, out='int')
    other_ctx = nufhe_b200.Context(rng=DeterministicRNG(5), thread=thr)
    other_sk = other_ctx.make_secret_key()
    other_ck, other_tk = other_ctx.make_cloud_key(other_sk, tree_key=True)
    other_tk.params = nufhe_b200.NuFHEParameters(tlwe_mask_size=2)
    with pytest.raises(ValueError, match='other parameters'):
        vm.make_encrypted_table(other_tk, x, out='bool')


def test_noise_functions():
    """rounding 9.9e-9, packing 3.03e-7 (DESIGN.md section 12's figure); a packed gate output read at m = 20 carries
    about 1.7e-5 after the key switch, and every configuration of lut.ALLOWED still keeps 7 sigma on it"""
    params = nufhe_b200.NuFHEParameters()
    assert IL.rounding_variance(params) == pytest.approx(9.95e-9, rel=0.01)
    assert IL.packing_variance(params) == pytest.approx(3.03e-7, rel=0.01)
    leaf = lut.bootstrap_variance(params) + IL.packing_variance(params)
    assert leaf + IL.output_variance(params, 20) == pytest.approx(1.72e-5, rel=0.01)
    for P, L, shift in lut.ALLOWED:
        assert 2.0**-(P + 2) / IL.lut_input_sigma(params, leaf, 20, L, shift) >= lut.MARGIN_SIGMAS, (P, L, shift)
        assert IL.lut_input_sigma(params, IL.rounding_variance(params), 20, L, shift) == lut.lut_sigma(params, L, shift)
    # the tightest: two 2-bit inputs x * 2 + y at two outputs per bootstrap
    assert 2.0**-4 / IL.lut_input_sigma(params, leaf, 20, 1, 0) == pytest.approx(7.9, abs=0.1)


def test_server_packed_table(env):
    """gate outputs packed under S with the tree key (packing.pack with the tree key's spectra), read back by index
    and fed to a gate: results decrypt to the gate outputs and record their variance plus packing and lookup"""
    ctx, thr = env['ctx'], env['thr']
    vm, ik, sk, tk = env['vms'][0], env['iks'][0], env['sks'][0], env['tks'][0]
    rng = numpy.random.RandomState(7)
    p, q = rng.randint(0, 2, size=(2, 8)).astype(bool)
    col = vm.gate_nand(ctx.encrypt(sk, p), ctx.encrypt(sk, q))
    t = vm.make_encrypted_table(tk, col, out='bool')
    assert (t.bits, t.columns, t.single, t.out) == (3, 1, True, 'bool')
    assert numpy.array_equal(t.data.numpy(), packing.pack(thr, tk, col).data.numpy())
    assert float(col.current_variances.max()) < lut.bootstrap_variance(sk.params)     # the key switch's only
    assert t.variance == pytest.approx(lut.bootstrap_variance(sk.params) + IL.packing_variance(sk.params))
    vals = numpy.array([0, 7, 3])
    r = vm.lookup(ctx.encrypt_index(ik, vals, 3), t)
    assert (ctx.decrypt(sk, r) == ~(p & q)[vals]).all()
    assert (ctx.decrypt(sk, vm.gate_nand(r, r)) == (p & q)[vals]).all()
    t2 = vm.make_encrypted_table(tk, [col, vm.gate_not(col)], out='bool')
    r2 = vm.lookup(ctx.encrypt_index(ik, vals, 3), t2)
    assert (ctx.decrypt(sk, r2[1]) == (p & q)[vals]).all()


@pytest.fixture(scope='module')
def mk_env(env):
    ctx, ik, cpk = env['ctx'], env['iks'], env['cpks']
    order = [0, 1, 0, 1]           # key 0, key 1, key 0 again, key 1 idle
    machine = ctx.make_multi_key_machine([env['cks'][k] for k in order])
    return dict(env, order=order, machine=machine)


@pytest.mark.parametrize('m, W', [(2, 1), (3, 2), (11, 1)])
def test_multikey_per_tenant_tables(mk_env, monkeypatch, m, W):
    """one encrypted table per tenant (one tenant idle): every tenant's results equal its own vm.lookup bit for bit,
    with the indirect level taking each query's table, in one pass and in passes of one query"""
    ctx, thr, machine, vms, iks, sks, order = (mk_env[k] for k in ('ctx', 'thr', 'machine', 'vms', 'iks', 'sks', 'order'))
    rng = numpy.random.RandomState(m * 3 + W)
    entries = [rng.randint(0, 4, size=(W, 1 << m)) for _ in range(3)]
    shape = lambda e: e if W > 1 else e[0]
    tables = [ctx.encrypt_table(iks[order[t]] if t != 1 else mk_env['cpks'][1], shape(entries[t]), bits=2)
              for t in range(3)] + [None]
    vals = [rng.randint(0, 1 << m, size=2), rng.randint(0, 1 << m, size=(1,)), rng.randint(0, 1 << m, size=(2, 1)), None]
    idx = [None if v is None else ctx.encrypt_index(iks[order[t]], v, m) for t, v in enumerate(vals)]
    for per_pass in (None, 1):
        if per_pass:
            monkeypatch.setattr(IL, 'queries_per_pass', lambda *a: per_pass)
        thr.indirect.clear()
        out = machine.lookup(idx, tables)
        assert out[3] is None
        kinds = {k for k, _, _ in thr.indirect}
        assert kinds == {'cmux' if m > 10 else 'rotate'}
        if per_pass is None:
            assert len(thr.indirect) == 1 and list(thr.indirect[0][2]) == [0, 0, 1, 2, 2]
        for t in range(3):
            want = vms[order[t]].lookup(idx[t], tables[t])
            got, want = ([out[t]], [want]) if W == 1 else (out[t], want)
            assert len(got) == W and all(_same(g, w) for g, w in zip(got, want)), (per_pass, t)
            for w in range(W):
                assert (ctx.decrypt_int(sks[order[t]], got[w], 2) == entries[t][w][vals[t]]).all(), (t, w)


def test_multikey_shared_table_and_errors(mk_env):
    """a repeated table is uploaded once per pass; a shared IndexTable still takes the direct levels; argument errors
    name the tenant"""
    ctx, thr, machine, vms, iks, order = (mk_env[k] for k in ('ctx', 'thr', 'machine', 'vms', 'iks', 'order'))
    t0 = ctx.encrypt_table(iks[0], numpy.arange(4), bits=2)
    idx = [ctx.encrypt_index(iks[order[t]], [t % 4], 2) for t in range(4)]
    thr.indirect.clear()
    out = machine.lookup(idx, [t0] * 4)
    assert thr.indirect[0][1] == 1 and list(thr.indirect[0][2]) == [0, 0, 0, 0]
    for t in range(4):
        assert _same(out[t], vms[order[t]].lookup(idx[t], t0))
    thr.indirect.clear()
    plain = vms[0].make_index_table(numpy.arange(4), bits=2)
    out = machine.lookup(idx, plain)
    assert not thr.indirect and all(_same(out[t], vms[order[t]].lookup(idx[t], plain)) for t in range(4))
    with pytest.raises(TypeError, match='tenant 2'):
        machine.lookup(idx, [t0, t0, plain, t0])
    with pytest.raises(TypeError, match='tenant 1'):
        machine.lookup(idx, [t0, None, t0, t0])
    with pytest.raises(ValueError, match='tenant 1.*share'):
        machine.lookup(idx, [t0, ctx.encrypt_table(iks[1], numpy.arange(8) % 4, bits=2), t0, t0])
    with pytest.raises(ValueError, match='one per tenant'):
        machine.lookup(idx, [t0])
    assert machine.lookup([None] * 4, [None] * 4) == [None] * 4


def test_multikey_rounds_on_compressed_keys():
    """resident_tenants = 2 with 3 active tenants: the tables go through the rounds with the indexes"""
    thr = EncryptedTableFakeEngine()
    ctx = nufhe_b200.Context(rng=DeterministicRNG(20261020), thread=thr)
    sks, cks, iks = [], [], []
    for _ in range(3):
        sk = ctx.make_secret_key()
        ck, ik = ctx.make_cloud_key(sk, compressed=True, index_key=True)
        sks.append(sk), cks.append(ck), iks.append(ik)
    machine = ctx.make_multi_key_machine(cks, resident_tenants=2)
    vms = [ctx.make_virtual_machine(ck.decompress(thr)) for ck in cks]
    tables = [ctx.encrypt_table(iks[t], (numpy.arange(8) + t) % 4, bits=2) for t in range(3)]
    vals = [numpy.array([1, 6]), numpy.array([7]), numpy.array([0, 3, 5])]
    idx = [ctx.encrypt_index(iks[t], v, 3) for t, v in enumerate(vals)]
    thr.indirect.clear()
    out = machine.lookup(idx, tables)
    assert len(thr.indirect) == 2 and [x[1] for x in thr.indirect] == [2, 1]
    for t in range(3):
        assert _same(out[t], vms[t].lookup(idx[t], tables[t])), t
        assert (ctx.decrypt_int(sks[t], out[t], 2) == ((numpy.arange(8) + t) % 4)[vals[t]]).all()
