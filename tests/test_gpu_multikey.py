"""The multi-key entry points (nb_mk_*, DESIGN.md section 17) against the single-key ones and the CPU oracle.

Every tenant's segment of a multi-key call must equal the single-key call on that segment with that tenant's key, bit
for bit (a, b and the key-switch variances), and small mixes must equal the oracle.  Outputs sit inside sentinel guard
rows.  Tenants cycle through three keys, so neighbouring tenants -- the two slots of a CTA, a chain resumed by another
CTA, two key-switch tiles -- always have different keys.  The mixes put tenant boundaries inside CTAs, run more chains
than resident CTAs in the default schedule and with forced chunk counts (chains resumed on other CTAs), and put a
tensor-core GEMM tenant and gather tenants in one key switch."""
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
SMALL_MIXES = [(1,), (1, 1), (1, 2, 3), (3, 0, 2, 1)]


@pytest.fixture(scope='module')
def oracle_keys():
    return [O.OracleKeys(20261017 + i) for i in range(KEYS)]


class Setup:
    def __init__(self, keys):
        from nufhe_b200.engine import Engine
        self.eng = eng = Engine(0)
        self.keys = keys
        self.bk = [eng.bk_prepare(eng.to_device(k.bk)) for k in keys]
        self.ks = [tuple(eng.to_device(x) for x in k.ks) for k in keys]


def make_setup(monkeypatch, keys, chunks=None):
    monkeypatch.delenv('NUFHE_B200_FORCE_CHUNKS', raising=False)
    if chunks:
        monkeypatch.setenv('NUFHE_B200_FORCE_CHUNKS', str(chunks))
    return Setup(keys)


@pytest.fixture(scope='module')
def default_setup(oracle_keys):
    return Setup(oracle_keys)


def segments(counts):
    lo = 0
    for t, c in enumerate(counts):
        yield t, lo, lo + c
        lo += c


def lwe(eng, rng, B, n):
    return (eng.to_device(rng.randint(-2**31, 2**31, size=(B, n), dtype=numpy.int32)),
            eng.to_device(rng.randint(-2**31, 2**31, size=(B,), dtype=numpy.int32)))


def rows(x, lo, hi):
    return None if x is None else (x[0][lo:hi], x[1][lo:hi])


def ptr(x):
    return None if x is None else ctypes.c_void_p(x.data_ptr())


def host(ctype, values):
    return (ctype * max(len(values), 1))(*values)


def guarded(eng, r, width):
    return torch.full((r + 2 * GUARD, width), SENTINEL, dtype=torch.int32, device=eng.device)


def unguard(buf, what):
    h = buf.cpu().numpy()
    assert (h[:GUARD] == SENTINEL).all() and (h[-GUARD:] == SENTINEL).all(), 'a store outside the rows of ' + what
    return h[GUARD:-GUARD]


def key_of(t):
    return t % KEYS


def mk_extract(s, counts, x1, x2, c, s1, s2, mu):
    eng, B = s.eng, sum(counts)
    oa, ob = guarded(eng, B, N), guarded(eng, B, 1)
    bks = host(ctypes.c_void_p, [s.bk[key_of(t)].data_ptr() for t in range(len(counts))])
    eng._call('nb_mk_bootstrap_extract', ptr(x1[0]), ptr(x1[1]), *(ptr(v) for v in (x2 or (None, None))), c, s1, s2,
              mu, bks, host(ctypes.c_size_t, counts), len(counts), 500, ptr(oa[GUARD:]), ptr(ob[GUARD:]), B)
    return unguard(oa, 'out_a'), unguard(ob, 'out_b')[:, 0]


def mk_keyswitch(s, counts, src1, src2, c):
    eng, B = s.eng, sum(counts)
    ra, rb = guarded(eng, B, 500), guarded(eng, B, 1)
    rcv = torch.full((B + 2 * GUARD,), -1.0, dtype=torch.float32, device=eng.device)
    T = len(counts)
    ks = [host(ctypes.c_void_p, [s.ks[key_of(t)][i].data_ptr() for t in range(T)]) for i in range(3)]
    eng._call('nb_mk_keyswitch', ptr(src1[0]), ptr(src1[1]), *(ptr(v) for v in (src2 or (None, None))), c, *ks,
              host(ctypes.c_size_t, counts), T, 1024, 500, 8, 2, ptr(ra[GUARD:]), ptr(rb[GUARD:]), ptr(rcv[GUARD:]), B)
    cv = rcv.cpu().numpy()
    assert (cv[:GUARD] == -1).all() and (cv[-GUARD:] == -1).all(), 'a store outside the rows of res_cv'
    return unguard(ra, 'res_a'), unguard(rb, 'res_b')[:, 0], cv[GUARD:-GUARD]


def check_gate(s, counts, seed, with_oracle):
    eng = s.eng
    rng = numpy.random.RandomState(seed)
    B = sum(counts)
    x1, x2 = lwe(eng, rng, B, 500), lwe(eng, rng, B, 500)
    c, s1, s2, mu = O.phase_to_t32(1, 8), -1, -1, O.MU
    got = mk_extract(s, counts, x1, x2, c, s1, s2, mu)
    for t, lo, hi in segments(counts):
        if hi == lo:
            continue
        wa, wb = eng.bootstrap_extract(rows(x1, lo, hi), rows(x2, lo, hi), c, s1, s2, mu, s.bk[key_of(t)])
        assert (got[0][lo:hi] == eng.to_host(wa)).all() and (got[1][lo:hi] == eng.to_host(wb)).all(), (counts, t)
        if with_oracle:
            a = (s1 * eng.to_host(x1[0][lo:hi]).astype(numpy.int64) + s2 * eng.to_host(x2[0][lo:hi]).astype(numpy.int64))
            b = c + s1 * eng.to_host(x1[1][lo:hi]).astype(numpy.int64) + s2 * eng.to_host(x2[1][lo:hi]).astype(numpy.int64)
            wrap = lambda v: (v & 0xffffffff).astype(numpy.uint32).view(numpy.int32)
            oa, ob = O.bootstrap(wrap(a), wrap(b), s.keys[key_of(t)].bk, None, mu)
            assert (got[0][lo:hi] == oa).all() and (got[1][lo:hi] == ob).all(), (counts, t)
    return x1


def check_keyswitch(s, counts, seed, fold, with_oracle):
    eng = s.eng
    rng = numpy.random.RandomState(seed)
    B = sum(counts)
    src1 = lwe(eng, rng, B, 1024)
    src2 = lwe(eng, rng, B, 1024) if fold else None
    c = O.phase_to_t32(1, 8) if fold else 0
    got = mk_keyswitch(s, counts, src1, src2, c)
    for t, lo, hi in segments(counts):
        if hi == lo:
            continue
        wa, wb, wcv = eng.keyswitch(s.ks[key_of(t)], rows(src1, lo, hi), rows(src2, lo, hi), c=c, want_cv=True)
        assert (got[0][lo:hi] == eng.to_host(wa)).all() and (got[1][lo:hi] == eng.to_host(wb)).all(), (counts, t)
        assert (got[2][lo:hi].view(numpy.uint32) == eng.to_host(wcv).view(numpy.uint32)).all(), (counts, t)
        if with_oracle:
            a = eng.to_host(src1[0][lo:hi]).astype(numpy.int64)
            b = eng.to_host(src1[1][lo:hi]).astype(numpy.int64) + c
            if fold:
                a = a + eng.to_host(src2[0][lo:hi]); b = b + eng.to_host(src2[1][lo:hi])
            wrap = lambda v: (v & 0xffffffff).astype(numpy.uint32).view(numpy.int32)
            oa, ob, _ = O.lwe_keyswitch(*s.keys[key_of(t)].ks, wrap(a), wrap(b))
            assert (got[0][lo:hi] == oa).all() and (got[1][lo:hi] == ob).all(), (counts, t)


@pytest.mark.parametrize('counts', SMALL_MIXES)
def test_small_mixes_gate_and_keyswitch(default_setup, counts):
    check_gate(default_setup, list(counts), 1, True)
    check_keyswitch(default_setup, list(counts), 2, False, True)
    check_keyswitch(default_setup, list(counts), 3, True, False)


@pytest.mark.parametrize('chunks', [None, 3, 5])
def test_700_single_ciphertext_tenants(monkeypatch, oracle_keys, chunks):
    s = make_setup(monkeypatch, oracle_keys, chunks)
    counts = [1] * 700
    check_gate(s, counts, 4, False)
    if chunks is None:
        check_keyswitch(s, counts, 5, True, False)


def test_gemm_and_gather_tenants_in_one_keyswitch(default_setup):
    s = default_setup
    planes = s.eng.ks_prepare(s.ks[0][0], s.ks[0][1])
    assert planes is not None
    try:
        check_keyswitch(s, [4096, 1], 6, False, False)
        check_keyswitch(s, [4096, 1, 3], 7, True, False)
    finally:
        s.eng.lib.nb_ks_forget(s.eng.handle, ctypes.c_void_p(s.ks[0][0].data_ptr()))


@pytest.mark.parametrize('counts', [(1, 2, 3), (3, 0, 2, 1)])
def test_extract2(default_setup, counts):
    s, eng = default_setup, default_setup.eng
    counts = list(counts)
    rng = numpy.random.RandomState(8)
    B = sum(counts)
    a, b, c = (lwe(eng, rng, B, 500) for _ in range(3))
    k1, k2 = O.phase_to_t32(-1, 8), O.phase_to_t32(-1, 8)
    oa, ob = guarded(eng, 2 * B, N), guarded(eng, 2 * B, 1)
    bks = host(ctypes.c_void_p, [s.bk[key_of(t)].data_ptr() for t in range(len(counts))])
    eng._call('nb_mk_bootstrap_extract2', ptr(a[0]), ptr(a[1]), ptr(b[0]), ptr(b[1]), k1, 1, 1, ptr(a[0]), ptr(a[1]),
              ptr(c[0]), ptr(c[1]), k2, -1, 1, O.MU, bks, host(ctypes.c_size_t, counts), len(counts), 500,
              ptr(oa[GUARD:]), ptr(ob[GUARD:]), B)
    ga, gb = unguard(oa, 'out_a'), unguard(ob, 'out_b')[:, 0]
    for t, lo, hi in segments(counts):
        if hi == lo:
            continue
        (u1a, u1b), (u2a, u2b) = eng.bootstrap_extract2((rows(a, lo, hi), rows(b, lo, hi), k1, 1, 1),
                                                        (rows(a, lo, hi), rows(c, lo, hi), k2, -1, 1), O.MU,
                                                        s.bk[key_of(t)])
        assert (ga[lo:hi] == eng.to_host(u1a)).all() and (gb[lo:hi] == eng.to_host(u1b)).all(), t
        assert (ga[B + lo:B + hi] == eng.to_host(u2a)).all() and (gb[B + lo:B + hi] == eng.to_host(u2b)).all(), t


@pytest.mark.parametrize('L', [0, 1, 2])
@pytest.mark.parametrize('two_inputs', [False, True])
def test_lut(default_setup, L, two_inputs):
    s, eng = default_setup, default_setup.eng
    counts = [1, 2, 0, 3]
    rng = numpy.random.RandomState(9 + L)
    B = sum(counts)
    x1 = lwe(eng, rng, B, 500)
    x2 = lwe(eng, rng, B, 500) if two_inputs else None
    tv = eng.to_device(rng.randint(-2**31, 2**31, size=(N,), dtype=numpy.int32))
    s1 = 4 if two_inputs else 1
    R = B << L
    oa, ob = guarded(eng, R, N), guarded(eng, R, 1)
    bks = host(ctypes.c_void_p, [s.bk[key_of(t)].data_ptr() for t in range(len(counts))])
    eng._call('nb_mk_bootstrap_lut_extract', ptr(x1[0]), ptr(x1[1]), *(ptr(v) for v in (x2 or (None, None))), 0, s1, 1,
              ptr(tv), 0, L, bks, host(ctypes.c_size_t, counts), len(counts), 500, ptr(oa[GUARD:]), ptr(ob[GUARD:]), B)
    ga, gb = unguard(oa, 'out_a'), unguard(ob, 'out_b')[:, 0]
    for t, lo, hi in segments(counts):
        if hi == lo:
            continue
        wa, wb = eng.bootstrap_lut_extract(rows(x1, lo, hi), rows(x2, lo, hi), 0, s1, 1, tv, L, s.bk[key_of(t)])
        assert (ga[lo << L:hi << L] == eng.to_host(wa)).all() and (gb[lo << L:hi << L] == eng.to_host(wb)).all(), t
    # the key switch of the 2^L samples of every ciphertext: counts * 2^L
    ks_counts = [c << L for c in counts]
    samples = (torch.from_numpy(ga).to(eng.device), torch.from_numpy(gb).to(eng.device))
    got = mk_keyswitch(s, ks_counts, samples, None, 0)
    for t, lo, hi in segments(ks_counts):
        if hi > lo:
            wa, wb, wcv = eng.keyswitch(s.ks[key_of(t)], rows(samples, lo, hi), want_cv=True)
            assert (got[0][lo:hi] == eng.to_host(wa)).all() and (got[1][lo:hi] == eng.to_host(wb)).all(), t


def test_refusals(monkeypatch, default_setup, oracle_keys):
    from nufhe_b200 import _native
    s, eng = default_setup, default_setup.eng
    lib = eng.lib
    x = lwe(eng, numpy.random.RandomState(10), 2, 500)
    out_a, out_b = eng.empty((2, N), torch.int32), eng.empty((2,), torch.int32)

    def extract(keys, counts, batch=2, n=500, e=eng):
        return lib.nb_mk_bootstrap_extract(e.handle, ptr(x[0]), ptr(x[1]), None, None, 0, 1, 0, O.MU,
                                           host(ctypes.c_void_p, keys), host(ctypes.c_size_t, counts), len(keys), n,
                                           ptr(out_a), ptr(out_b), batch)
    good = [s.bk[0].data_ptr(), s.bk[1].data_ptr()]
    assert extract(good, [1, 1]) == _native.NB_OK
    assert extract(good, [1, 0], batch=2) == _native.NB_EINVAL                       # counts do not add up
    assert extract([good[0], None], [1, 1]) == _native.NB_EINVAL                     # null key
    unregistered = eng.empty((500, eng.lib.nb_bk_row_u64()), torch.int64)
    assert extract([good[0], unregistered.data_ptr()], [1, 1]) == _native.NB_EINVAL
    assert 'tenant 1' in lib.nb_last_error(eng.handle).decode()
    mb = eng.bk_prepare_multibit(eng.to_device(oracle_keys[0].bk[:6]))
    assert extract([good[0], mb.data_ptr()], [1, 1]) == _native.NB_EUNSUPPORTED
    assert extract(good, [1, 1], n=0) == _native.NB_EUNSUPPORTED
    assert lib.nb_mk_bootstrap_extract(eng.handle, ptr(x[0]), ptr(x[1]), None, None, 0, 1, 0, O.MU, None,
                                       host(ctypes.c_size_t, [2]), 1, 500, ptr(out_a), ptr(out_b), 2) == _native.NB_EINVAL
    ks = [host(ctypes.c_void_p, [s.ks[0][i].data_ptr()]) for i in range(3)]
    src = lwe(eng, numpy.random.RandomState(11), 2, 1024)
    res_a, res_b = eng.empty((2, 500), torch.int32), eng.empty((2,), torch.int32)
    assert lib.nb_mk_keyswitch(eng.handle, ptr(src[0]), ptr(src[1]), None, None, 0, *ks, host(ctypes.c_size_t, [2]), 1,
                               1024, 499, 8, 2, ptr(res_a), ptr(res_b), None, 2) == _native.NB_EUNSUPPORTED
    assert lib.nb_mk_keyswitch(eng.handle, ptr(src[0]), ptr(src[1]), None, None, 0, *ks, host(ctypes.c_size_t, [3]), 1,
                               1024, 500, 8, 2, ptr(res_a), ptr(res_b), None, 2) == _native.NB_EINVAL
    # a context with the FP64 step disabled
    monkeypatch.setenv('NUFHE_B200_FFT', '0')
    from nufhe_b200.engine import Engine
    e0 = Engine(0)
    bk0 = e0.bk_prepare(e0.to_device(oracle_keys[0].bk))
    assert extract([bk0.data_ptr()], [2], e=e0) == _native.NB_EUNSUPPORTED


def test_api_matches_per_tenant_machines():
    import nufhe_b200 as nufhe
    ctx = nufhe.Context(rng=nufhe.DeterministicRNG(77))
    sks = [ctx.make_secret_key() for _ in range(3)]
    cks = [ctx.make_cloud_key(sk) for sk in sks[:2]]
    cks.append(ctx.make_cloud_key(sks[2], compressed=True).decompress(ctx.thread))
    # tenants: key 0, key 1, key 0 again, a decompressed compressed key, an idle tenant (key 1)
    tenant_keys = [0, 1, 0, 2, 1]
    machine = ctx.make_multi_key_machine([cks[k] for k in tenant_keys])
    vms = [ctx.make_virtual_machine(ck) for ck in cks]
    rng = numpy.random.RandomState(12)
    sizes = [5, 1, 3, 4, None]
    bits = [None if n is None else [rng.randint(0, 2, n).astype(bool) for _ in range(3)] for n in sizes]
    enc = [[None if b is None else ctx.encrypt(sks[tenant_keys[t]], b[i]) for t, b in enumerate(bits)] for i in range(3)]

    def same(x, y):
        return ((x.a == y.a).all() and (x.b == y.b).all() and (x.current_variances == y.current_variances).all()).item()

    for name, truth in (('nand', lambda a, b: ~(a & b)), ('xor', lambda a, b: a ^ b)):
        out = getattr(machine, 'gate_' + name)(enc[0], enc[1])
        assert out[4] is None
        for t in range(4):
            want = getattr(vms[tenant_keys[t]], 'gate_' + name)(enc[0][t], enc[1][t])
            assert same(out[t], want), (name, t)
            assert (ctx.decrypt(sks[tenant_keys[t]], out[t]) == truth(bits[t][0], bits[t][1])).all(), (name, t)
    out = machine.gate_mux(*enc)
    for t in range(4):
        assert same(out[t], vms[tenant_keys[t]].gate_mux(enc[0][t], enc[1][t], enc[2][t])), t
        assert (ctx.decrypt(sks[tenant_keys[t]], out[t]) == numpy.where(bits[t][0], bits[t][1], bits[t][2])).all(), t
    table = vms[0].make_lut([[v % 2 for v in range(4)], [v // 2 for v in range(4)]], bits=2)
    vals = [None if n is None else rng.randint(0, 4, n) for n in sizes]
    xs = [None if v is None else ctx.encrypt_int(sks[tenant_keys[t]], v, 2) for t, v in enumerate(vals)]
    out = machine.lut(table, xs)
    for t in range(4):
        want = vms[tenant_keys[t]].lut(table, xs[t])
        assert all(same(o, w) for o, w in zip(out[t], want)), t
        assert (ctx.decrypt_int(sks[tenant_keys[t]], out[t][0], 2) == vals[t] % 2).all(), t
        assert (ctx.decrypt_int(sks[tenant_keys[t]], out[t][1], 2) == vals[t] // 2).all(), t
    with pytest.raises(ValueError, match='tenant 1'):
        ctx.make_multi_key_machine([cks[0], ctx.make_cloud_key(sks[0], multi_bit=2)])
    with pytest.raises(TypeError, match='tenant 1'):
        ctx.make_multi_key_machine([cks[0], ctx.make_cloud_key(sks[1], compressed=True)])
