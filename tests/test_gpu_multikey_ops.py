"""The multi-key tree LUTs, packing, expansion, index lookups and per-tenant LUT tables (DESIGN.md section 18) on the GPU.

Through the C ABI, with outputs inside sentinel guard rows: every tenant's segment of nb_mk_tree_keyswitch,
nb_mk_bootstrap_glwe_lut_extract and nb_mk_ntt_mac equals the single-key call with that tenant's key, bit for bit.
Tenants cycle through three keys, so neighbouring tenants always have different keys; 700 single-ciphertext tenants run
more chains than resident CTAs.  Through Python, every operation of the multi-key machine equals per-tenant
VirtualMachines and decrypts to the truth table, with a decompressed compressed cloud key, a repeated key, an idle
tenant and pass boundaries."""
import ctypes

import numpy
import pytest
import torch

from oracle import oracle as O

pytestmark = pytest.mark.gpu
N = 1024
GUARD = 4
SENTINEL = -0x3c3c3c3d
KEYS = 3
MIXES = [(1,), (1, 1), (1, 2, 3), (3, 0, 2, 1), (1,) * 700]


def segments(counts):
    lo = 0
    for t, c in enumerate(counts):
        yield t, lo, lo + c
        lo += c


def ptr(x):
    return None if x is None else ctypes.c_void_p(x.data_ptr())


def host(ctype, values):
    return (ctype * max(len(values), 1))(*values)


def guarded(eng, shape, dtype=torch.int32, fill=SENTINEL):
    return torch.full((shape[0] + 2 * GUARD,) + tuple(shape[1:]), fill, dtype=dtype, device=eng.device)


def unguard(buf, what, fill=SENTINEL):
    h = buf.cpu().numpy()
    assert (h[:GUARD] == fill).all() and (h[-GUARD:] == fill).all(), 'a store outside the rows of ' + what
    return h[GUARD:-GUARD]


def rand_i32(rng, shape):
    return rng.randint(-2**31, 2**31, size=shape, dtype=numpy.int64).astype(numpy.int32)


@pytest.fixture(scope='module')
def oracle_keys():
    return [O.OracleKeys(20261018 + i) for i in range(KEYS)]


def engine(monkeypatch, chunks=None):
    from nufhe_b200.engine import Engine
    monkeypatch.delenv('NUFHE_B200_FORCE_CHUNKS', raising=False)
    if chunks:
        monkeypatch.setenv('NUFHE_B200_FORCE_CHUNKS', str(chunks))
    return Engine(0)


# ---------------------------------------------------------------- C ABI

@pytest.mark.parametrize('counts', MIXES, ids=lambda c: 'x'.join(map(str, c[:4])) + ('..' if len(c) > 4 else ''))
def test_tree_keyswitch(monkeypatch, counts):
    eng = engine(monkeypatch)
    rng = numpy.random.RandomState(len(counts))
    n, k = 500, 1
    planes = [eng.tree_prepare(eng.to_device(rand_i32(rng, (n, 2, k, N))), eng.to_device(rand_i32(rng, (n, 2, N))))
              for _ in range(KEYS)]
    counts = [c * 100 + (c > 1) * 57 for c in counts] if len(counts) < 5 else list(counts)   # tiles of 256 and remainders
    R = sum(counts)
    a = eng.to_device(rand_i32(rng, (R, n)))
    out = guarded(eng, (R, k + 1, N))
    eng._call('nb_mk_tree_keyswitch', ptr(a), host(ctypes.c_void_p, [planes[t % KEYS].data_ptr() for t in range(len(counts))]),
              host(ctypes.c_size_t, counts), len(counts), n, k, ptr(out[GUARD:]), R)
    got = unguard(out, 'out')
    for t, lo, hi in segments(counts):
        if hi > lo:
            assert (got[lo:hi] == eng.to_host(eng.tree_keyswitch(a[lo:hi], planes[t % KEYS], k))).all(), (counts[:4], t)


# forced chunk counts act when there are more chains than resident CTAs: with the 700 tenants
@pytest.mark.parametrize('counts,chunks', [(c, None) for c in MIXES] + [(MIXES[-1], 3), (MIXES[-1], 5)],
                         ids=lambda v: v if v is None or isinstance(v, int) else
                         'x'.join(map(str, v[:4])) + ('..' if len(v) > 4 else ''))
def test_bootstrap_glwe_lut_extract(monkeypatch, oracle_keys, counts, chunks):
    eng = engine(monkeypatch, chunks)
    bks = [eng.bk_prepare(eng.to_device(k.bk)) for k in oracle_keys]
    rng = numpy.random.RandomState(7 + len(counts))
    B = sum(counts)
    x = (eng.to_device(rand_i32(rng, (B, 500))), eng.to_device(rand_i32(rng, (B,))))
    tv = eng.to_device(rand_i32(rng, (B, 2, N)))
    oa, ob = guarded(eng, (B, N)), guarded(eng, (B,))
    eng._call('nb_mk_bootstrap_glwe_lut_extract', ptr(x[0]), ptr(x[1]), ptr(tv),
              host(ctypes.c_void_p, [bks[t % KEYS].data_ptr() for t in range(len(counts))]),
              host(ctypes.c_size_t, list(counts)), len(counts), 500, ptr(oa[GUARD:]), ptr(ob[GUARD:]), B)
    ga, gb = unguard(oa, 'out_a'), unguard(ob, 'out_b')
    for t, lo, hi in segments(counts):
        if hi > lo:
            wa, wb = eng.bootstrap_glwe_lut_extract((x[0][lo:hi], x[1][lo:hi]), tv[lo:hi], bks[t % KEYS])
            assert (ga[lo:hi] == eng.to_host(wa)).all() and (gb[lo:hi] == eng.to_host(wb)).all(), (counts[:4], t)


@pytest.mark.parametrize('counts', MIXES, ids=lambda c: 'x'.join(map(str, c[:4])) + ('..' if len(c) > 4 else ''))
def test_ntt_mac(monkeypatch, counts):
    eng = engine(monkeypatch)
    rng = numpy.random.RandomState(11 + len(counts))
    R, U = 6, 3
    G = sum(counts)
    p = numpy.uint64(O.P)
    field = lambda shape: eng.to_device(rng.randint(0, 2**63, size=shape, dtype=numpy.int64).view(numpy.uint64) % p)
    keys = [field((R, U, N)) for _ in range(KEYS)]
    x = field((G, R, N))
    out = guarded(eng, (G, U, N), torch.int64, -1)
    eng._call('nb_mk_ntt_mac', ptr(x), host(ctypes.c_void_p, [keys[t % KEYS].data_ptr() for t in range(len(counts))]),
              host(ctypes.c_size_t, list(counts)), len(counts), ptr(out[GUARD:]), R, U, G)
    got = unguard(out, 'out', -1)
    for t, lo, hi in segments(counts):
        if hi > lo:
            assert (got[lo:hi] == eng.to_host(eng.ntt_mac(x[lo:hi], keys[t % KEYS]))).all(), (counts[:4], t)


def test_refusals(monkeypatch, oracle_keys):
    from nufhe_b200 import _native
    eng = engine(monkeypatch)
    lib = eng.lib
    rng = numpy.random.RandomState(3)
    planes = eng.tree_prepare(eng.to_device(rand_i32(rng, (500, 2, 1, N))), eng.to_device(rand_i32(rng, (500, 2, N))))
    a = eng.to_device(rand_i32(rng, (2, 500)))
    out = eng.empty((2, 2, N), torch.int32)

    def tree(pl, counts, n=500):
        return lib.nb_mk_tree_keyswitch(eng.handle, ptr(a), host(ctypes.c_void_p, pl), host(ctypes.c_size_t, counts),
                                        len(pl), n, 1, ptr(out), 2)
    assert tree([planes.data_ptr()] * 2, [1, 1]) == _native.NB_OK
    assert tree([planes.data_ptr()] * 2, [1, 2]) == _native.NB_EINVAL
    assert tree([planes.data_ptr(), None], [1, 1]) == _native.NB_EINVAL
    assert 'tenant 1' in lib.nb_last_error(eng.handle).decode()
    assert tree([planes.data_ptr()], [2], n=0) == _native.NB_EINVAL
    bk = eng.bk_prepare(eng.to_device(oracle_keys[0].bk))
    x = (eng.to_device(rand_i32(rng, (2, 500))), eng.to_device(rand_i32(rng, (2,))))
    tv = eng.to_device(rand_i32(rng, (2, 2, N)))
    oa, ob = eng.empty((2, N), torch.int32), eng.empty((2,), torch.int32)

    def glwe(keys, counts):
        return lib.nb_mk_bootstrap_glwe_lut_extract(eng.handle, ptr(x[0]), ptr(x[1]), ptr(tv), host(ctypes.c_void_p, keys),
                                                    host(ctypes.c_size_t, counts), len(keys), 500, ptr(oa), ptr(ob), 2)
    assert glwe([bk.data_ptr()], [2]) == _native.NB_OK
    assert glwe([bk.data_ptr()], [1]) == _native.NB_EINVAL
    unregistered = eng.empty((500, lib.nb_bk_row_u64()), torch.int64)
    assert glwe([bk.data_ptr(), unregistered.data_ptr()], [1, 1]) == _native.NB_EINVAL
    mb = eng.bk_prepare_multibit(eng.to_device(oracle_keys[0].bk[:6]))
    assert glwe([bk.data_ptr(), mb.data_ptr()], [1, 1]) == _native.NB_EUNSUPPORTED
    key = eng.empty((4, 2, N), torch.int64).zero_()
    xs = eng.empty((2, 4, N), torch.int64).zero_()
    mo = eng.empty((2, 2, N), torch.int64)

    def mac(keys, counts, rows=4):
        return lib.nb_mk_ntt_mac(eng.handle, ptr(xs), host(ctypes.c_void_p, keys), host(ctypes.c_size_t, counts),
                                 len(keys), ptr(mo), rows, 2, 2)
    assert mac([key.data_ptr()] * 2, [1, 1]) == _native.NB_OK
    assert mac([key.data_ptr()] * 2, [2, 1]) == _native.NB_EINVAL
    assert mac([key.data_ptr(), None], [1, 1]) == _native.NB_EINVAL
    assert mac([key.data_ptr()], [2], rows=0) == _native.NB_EINVAL


# ---------------------------------------------------------------- Python

@pytest.fixture(scope='module')
def env():
    import nufhe_b200 as nufhe
    ctx = nufhe.Context(rng=nufhe.DeterministicRNG(20261019))
    sks, cks, tks, iks, cpks, pks, psks = [], [], [], [], [], [], []
    for i in range(3):
        sk = ctx.make_secret_key()
        ck, tk, ik, cpk = ctx.make_cloud_key(sk, compressed=(i == 2), tree_key=True, index_key=True,
                                             compact_public_key=True)
        if i == 2:
            ck = ck.decompress(ctx.thread)
        psk, pk = ctx.make_packing_keys(sk)
        for lst, v in zip((sks, cks, tks, iks, cpks, pks, psks), (sk, ck, tk, ik, cpk, pk, psk)):
            lst.append(v)
    # tenants: key 0, key 1, key 0 again, the decompressed compressed key, an idle tenant (key 1)
    order = [0, 1, 0, 2, 1]
    return dict(nufhe=nufhe, ctx=ctx, sks=sks, cks=cks, tks=tks, iks=iks, cpks=cpks, pks=pks, psks=psks, order=order,
                machine=ctx.make_multi_key_machine([cks[k] for k in order]), vms=[ctx.make_virtual_machine(c) for c in cks])


def same(x, y):
    return (tuple(x.shape) == tuple(y.shape) and (x.a == y.a).all() and (x.b == y.b).all()
            and (x.current_variances == y.current_variances).all()).item()


SIZES = [3, 1, 2, 4, None]


@pytest.mark.parametrize('bits,D', [(1, 2), (1, 3), (2, 2), (2, 3)])
def test_lut_tree(env, bits, D):
    ctx, machine, sks, vms, tks, order = (env[k] for k in ('ctx', 'machine', 'sks', 'vms', 'tks', 'order'))
    M = 1 << bits
    rng = numpy.random.RandomState(bits * 10 + D)
    tables = rng.randint(0, M, size=(3,) + (M,) * D)            # three functions
    table = vms[0].make_tree_lut(tables, bits, D)
    vals = [None if s is None else rng.randint(0, M, size=(D, s)) for s in SIZES]
    digits = [[None if v is None else ctx.encrypt_int(sks[order[t]], v[i], bits) for t, v in enumerate(vals)]
              for i in range(D)]
    out = machine.lut_tree([tks[k] for k in order[:4]] + [None], table, digits)
    assert out[4] is None
    for t in range(4):
        want = vms[order[t]].lut_tree(tks[order[t]], table, [d[t] for d in digits])
        assert all(same(o, w) for o, w in zip(out[t], want)), (bits, D, t)
        for f in range(3):
            assert (ctx.decrypt_int(sks[order[t]], out[t][f], bits) == tables[(f,) + tuple(vals[t])]).all(), (t, f)


def test_lut_tree_pass_boundary(env, monkeypatch):
    from nufhe_b200 import tree_lut
    ctx, machine, sks, vms, tks, order = (env[k] for k in ('ctx', 'machine', 'sks', 'vms', 'tks', 'order'))
    table = vms[0].make_tree_lut(numpy.array([[0, 1], [1, 0]]), 1, 2, out='bool')
    monkeypatch.setattr(tree_lut, 'ROWS_PER_PASS', 2 * table.groups)             # two ciphertexts per pass
    rng = numpy.random.RandomState(5)
    vals = [None if s is None else rng.randint(0, 2, size=(2, s)) for s in SIZES]
    digits = [[None if v is None else ctx.encrypt_int(sks[order[t]], v[i], 1) for t, v in enumerate(vals)]
              for i in range(2)]
    out = machine.lut_tree([tks[k] for k in order], table, digits)
    for t in range(4):
        assert same(out[t], vms[order[t]].lut_tree(tks[order[t]], table, [d[t] for d in digits])), t
        assert (ctx.decrypt(sks[order[t]], out[t]) == (vals[t][0] ^ vals[t][1]).astype(bool)).all(), t


def test_lut_per_tenant_tables(env):
    ctx, machine, sks, vms, order = (env[k] for k in ('ctx', 'machine', 'sks', 'vms', 'order'))
    fs = [lambda v: (v + 1) % 4, lambda v: 3 - v, lambda v: v * v % 4, lambda v: v // 2]
    tables = [vms[0].make_lut([f(v) for v in range(4)], bits=2) for f in fs] + [None]
    rng = numpy.random.RandomState(6)
    vals = [None if s is None else rng.randint(0, 4, s) for s in SIZES]
    xs = [None if v is None else ctx.encrypt_int(sks[order[t]], v, 2) for t, v in enumerate(vals)]
    out = machine.lut(tables, xs)
    assert out[4] is None
    for t in range(4):
        assert same(out[t], vms[order[t]].lut(tables[t], xs[t])), t
        assert (ctx.decrypt_int(sks[order[t]], out[t], 2) == fs[t](vals[t])).all(), t


def test_pack(env):
    ctx, machine, sks, vms, pks, psks, order = (env[k] for k in ('ctx', 'machine', 'sks', 'vms', 'pks', 'psks', 'order'))
    rng = numpy.random.RandomState(7)
    sizes = [3, 1025, None, 1024, 2]
    bits = [None if s is None else rng.randint(0, 2, s).astype(bool) for s in sizes]
    cts = [None if b is None else ctx.encrypt(sks[order[t]], b) for t, b in enumerate(bits)]
    out = machine.pack([None if b is None else pks[order[t]] for t, b in enumerate(bits)], cts)
    assert out[2] is None
    for t in (0, 1, 3, 4):
        assert out[t] == vms[order[t]].pack(pks[order[t]], cts[t]), t
        assert (ctx.decrypt(psks[order[t]], out[t]) == bits[t]).all(), t


def test_expand_with_pass_boundary(env, monkeypatch):
    from nufhe_b200 import compact
    ctx, machine, sks, vms, cpks, order = (env[k] for k in ('ctx', 'machine', 'sks', 'vms', 'cpks', 'order'))
    rng = numpy.random.RandomState(8)
    sizes = [3, 1500, 1, None, 2]
    bits = [None if s is None else rng.randint(0, 2, s).astype(bool) for s in sizes]
    cs = [None if b is None else ctx.encrypt(cpks[order[t]], b) for t, b in enumerate(bits)]
    for per_pass in (None, 1):
        if per_pass:
            monkeypatch.setattr(compact, 'groups_per_pass', lambda params: per_pass)
        out = machine.expand(cs)
        assert out[3] is None
        for t in (0, 1, 2, 4):
            assert same(out[t], vms[order[t]].expand(cs[t])), (per_pass, t)
            assert (ctx.decrypt(sks[order[t]], out[t]) == bits[t]).all(), (per_pass, t)


@pytest.mark.parametrize('m,W', [(8, 4), (16, 1)])
def test_lookup_with_pass_boundary(env, monkeypatch, m, W):
    from nufhe_b200 import index_lookup
    ctx, machine, sks, vms, iks, order = (env[k] for k in ('ctx', 'machine', 'sks', 'vms', 'iks', 'order'))
    rng = numpy.random.RandomState(m + W)
    entries = rng.randint(0, 4, size=(W, 1 << m))
    table = vms[0].make_index_table(entries if W > 1 else entries[0], bits=2)
    vals = [None if s is None else rng.randint(0, 1 << m, s) for s in SIZES]
    idx = [None if v is None else ctx.encrypt_index(iks[order[t]], v, m) for t, v in enumerate(vals)]
    for per_pass in (None, 3):
        if per_pass:
            monkeypatch.setattr(index_lookup, 'queries_per_pass', lambda m_, w_: per_pass)
        out = machine.lookup(idx, table)
        assert out[4] is None
        for t in range(4):
            want = vms[order[t]].lookup(idx[t], table)
            got, want = ([out[t]], [want]) if W == 1 else (out[t], want)
            assert all(same(g, w) for g, w in zip(got, want)), (per_pass, t)
            for w in range(W):
                assert (ctx.decrypt_int(sks[order[t]], got[w], 2) == entries[w][vals[t]]).all(), (t, w)
