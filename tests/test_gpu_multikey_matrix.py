"""Every multi-key entry point (nb_mk_*, DESIGN.md sections 17 and 18) in every schedule, dimension and key-switch
split, bit for bit against the exact CPU oracle (tests/mk_ref.py, fused_ref.py, ks_ref.py, tree_ref.py).

Every call goes through the C ABI with its outputs inside buffers whose guard rows must keep their sentinel.  Tenants
cycle through three keys, so neighbouring tenants -- the two slots of a CTA, the last ciphertext of extract2's job A and
the first of job B, a chain resumed by another CTA, two key-switch or tree tiles -- always have different keys.

Bootstrap at n = 25: the modes of tests/test_gpu_fused_matrix.py with edge rows first, each on one of three tenant
layouts (one tenant; one ciphertext per tenant; a mix with idle tenants first, in the middle and last, and tenant
boundaries at both slot parities), at batches around one wave W of BrFftMk (2 CTAs per SM, 2 ciphertexts each), in
the default schedule, without the start-up stagger (single waves), with one chunk per chain and 4 forced chunks
(multi-wave: at n = 25 chains resume on odd steps on other CTAs), and under each forced shape setting of the single-key
launch, which the multi-key launch must ignore.  A batch's layout is the first B rows of the mode's layout on its
largest batch, so the oracle runs once per mode.  Every cell repeats the largest batch of each mode with tenant 1's key
spoiled (its FP64 part zeroed): every other tenant's rows must keep the oracle's bits, tenant 1's must change unless the
mode is key-free.  n = 500: NAND on real encryptions under each tenant's key, key-switched and decrypted per tenant,
extract2, LUT and GLWE.  n = 1024 and n = 1: three single-ciphertext tenants.

nb_mk_keyswitch at both edges of every split band of its gather kernel, at segments of 31, 32 and 33 rows, with a GEMM
tenant at the engine's threshold and one below it in split 1 and split > 1 launches, with and without the fold and
res_cv, an edge key and edge rows; variances must equal the fixed-shape float32 sum bit for bit.  nb_mk_tree_keyswitch
at tile edges for k = 1, 2 and n = 500, 25, 1, and at the exactness bound.  nb_mk_ntt_mac with field elements at p - 1
and two output tiles against Python-integer arithmetic."""
import ctypes
import functools

import numpy
import pytest
import torch

import fused_ref as F
import gen_inputs as G
import ks_ref as K
import mk_ref as MK
import tree_ref
from fused_ref import gate_mode, glwe_mode, lut_mode, x2_mode
from oracle import oracle as O

pytestmark = pytest.mark.gpu
N = 1024
KEYS = 3
FFT_U64 = 16 * 512 * 2                      # the FP64 part at the end of every engine key row
SPOILED = 1                                 # the tenant whose key is spoiled in the repeat of each cell

# the single-key launch's shape settings (WIDE_MAX, WIDE2_MAX, PAIR_MAX, PAIR_ASYNC), which the multi-key launch ignores
SHAPE_ENV = ('NUFHE_B200_WIDE_MAX', 'NUFHE_B200_WIDE2_MAX', 'NUFHE_B200_PAIR_MAX', 'NUFHE_B200_PAIR_ASYNC')
SHAPES = {'default': None, 'wide': ('1000000', '0', '0', '1'), 'wide2': ('1000000', '1000000', '0', '1'),
          'pair': ('0', '0', '1000000', '1'), 'pair_barrier': ('0', '0', '1000000', '0')}
SCHEDULES = {'default': {}, 'stagger0': {'NUFHE_B200_STAGGER': '0'}, 'one_chunk': {'NUFHE_B200_MAX_CHUNKS': '1'},
             'force4': {'NUFHE_B200_FORCE_CHUNKS': '4'}}
CELLS = ([('default', s) for s in SCHEDULES] + [(s, 'default') for s in SHAPES if s != 'default'])


@functools.lru_cache(None)
def sm_count():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def W():
    return MK.wave(sm_count())


def engine(monkeypatch, shape='default', schedule='default', extra=None):
    from nufhe_b200.engine import Engine
    for k in list(SHAPE_ENV) + ['NUFHE_B200_FFT', 'NUFHE_B200_KS_MMA_MIN'] + [k for s in SCHEDULES.values() for k in s]:
        monkeypatch.delenv(k, raising=False)
    for k, v in zip(SHAPE_ENV, SHAPES[shape] or ()):
        monkeypatch.setenv(k, v)
    for k, v in list(SCHEDULES[schedule].items()) + list((extra or {}).items()):
        monkeypatch.setenv(k, v)
    return Engine()


def host(ctype, values):
    return (ctype * max(len(values), 1))(*values)


def sizes_t(counts):
    return host(ctypes.c_size_t, [int(c) for c in counts])


# ---- layouts --------------------------------------------------------------------------------------------------------

MIX_PATTERN = (3, 1, 0, 2, 5, 4, 0, 1, 7, 6, 2, 9)      # idle tenants inside; boundaries at odd and even rows


def layout(kind, M):
    """a count list of M rows: 'one' tenant, 'ones' (every tenant one ciphertext, so every CTA holds two tenants) or
    'mixed' (an idle tenant first, MIX_PATTERN repeated, an idle tenant last)"""
    if kind == 'one':
        return [M]
    if kind == 'ones':
        return [1] * M
    counts, left, i = [0], M, 0
    while left:
        c = min(MIX_PATTERN[i % len(MIX_PATTERN)], left)
        counts.append(c)
        left -= c
        i += 1
    return counts + [0]


LAYOUTS = ('mixed', 'ones', 'one')


class Keys:
    """every tenant's engine key on one engine (tenant t: key t % 3), and each key prepared again with its FP64 part
    zeroed (it stays registered), for the tenant whose key is spoiled"""

    def __init__(self, eng, bks):
        self.bk = [eng.bk_prepare(eng.to_device(k)) for k in bks]
        self.spoiled = [eng.bk_prepare(eng.to_device(k)) for k in bks]
        for s in self.spoiled:
            s[:, -FFT_U64:] = 0

    def ptrs(self, tenants, spoil=None):
        return host(ctypes.c_void_p, [(self.spoiled if t == spoil else self.bk)[t % KEYS].data_ptr()
                                      for t in range(tenants)])


# ---- the modes of fused_ref with their multi-key calls --------------------------------------------------------------
# A mode's `call(eng, dev, run, b)` takes run = (Keys, the mode's layout on its largest batch, the spoiled tenant or
# None); the call's counts are the first b rows of that layout.

def _bks(run, b):
    keys, master, spoil = run
    counts = MK.truncate(master, b)
    return keys.ptrs(len(counts), spoil), sizes_t(counts), len(counts)


def _outs(eng, rows):
    return F.guarded(eng, rows, N), F.guarded(eng, rows, 1)


def mk_gate(name, n, bks, c, s1, s2, mu, two, seed, B, master, rows=None, x=None):
    m = gate_mode(name, n, per_tenant(bks, master), c, s1, s2, mu, two, seed, B, rows, x, ref=_ref(master, rows, B))

    def call(eng, dev, run, b):
        (a1, b1), (a2, b2) = dev
        oa, ob = _outs(eng, b)
        eng._call('nb_mk_bootstrap_extract', F.ptr(a1), F.ptr(b1), F.ptr(a2), F.ptr(b2), c, s1, s2, mu,
                  *_bks(run, b), n, oa[F.GUARD].data_ptr(), ob[F.GUARD].data_ptr(), b)
        return F.unguard(oa, 'out_a'), F.unguard(ob, 'out_b')[:, 0]
    m.call, m.master = call, master
    return m


def mk_x2(name, n, bks, job_a, job_b, mu, seed, B, master, rows=None):
    m = x2_mode(name, n, per_tenant(bks, master), job_a, job_b, mu, seed, B, rows, ref=_ref(master, rows, B))

    def call(eng, dev, run, b):
        (a1, b1), (a2, b2), (c1, d1), (c2, d2) = dev
        oa, ob = _outs(eng, 2 * b)
        eng._call('nb_mk_bootstrap_extract2', F.ptr(a1), F.ptr(b1), F.ptr(a2), F.ptr(b2), *job_a[:3],
                  F.ptr(c1), F.ptr(d1), F.ptr(c2), F.ptr(d2), *job_b[:3], mu, *_bks(run, b), n,
                  oa[F.GUARD].data_ptr(), ob[F.GUARD].data_ptr(), b)
        ga, gb = F.unguard(oa, 'out_a'), F.unguard(ob, 'out_b')[:, 0]
        return ga[:b], gb[:b], ga[b:], gb[b:]
    m.call, m.master = call, master
    return m


def mk_lut(name, n, bks, L, per_ct, two, seed, B, master, rows=None):
    m = lut_mode(name, n, per_tenant(bks, master), L, per_ct, two, seed, B, rows, ref=_ref(master, rows, B))
    c, s1, s2 = (12345678, 2, -3) if two else (-987654, -1, 5)       # lut_mode's constants
    K_ = 1 << L

    def call(eng, dev, run, b):
        (a1, b1), (a2, b2), dtv = dev
        oa, ob = _outs(eng, b * K_)
        eng._call('nb_mk_bootstrap_lut_extract', F.ptr(a1), F.ptr(b1), F.ptr(a2), F.ptr(b2), c, s1, s2, dtv.data_ptr(),
                  N if per_ct else 0, L, *_bks(run, b), n, oa[F.GUARD].data_ptr(), ob[F.GUARD].data_ptr(), b)
        return F.unguard(oa, 'out_a').reshape(b, K_, N), F.unguard(ob, 'out_b').reshape(b, K_)
    m.call, m.master = call, master
    return m


def mk_glwe(name, n, bks, seed, B, master, rows=None):
    m = glwe_mode(name, n, per_tenant(bks, master), seed, B, rows, ref=_ref(master, rows, B))

    def call(eng, dev, run, b):
        (a, bb), dtv = dev
        oa, ob = _outs(eng, b)
        eng._call('nb_mk_bootstrap_glwe_lut_extract', F.ptr(a), F.ptr(bb), dtv.data_ptr(), *_bks(run, b), n,
                  oa[F.GUARD].data_ptr(), ob[F.GUARD].data_ptr(), b)
        return F.unguard(oa, 'out_a'), F.unguard(ob, 'out_b')[:, 0]
    m.call, m.master = call, master
    return m


def per_tenant(bks, master):
    """the key of every tenant of a layout (tenant t: key t % 3), as mk_ref.ref takes them"""
    return [bks[t % KEYS] for t in range(len(master))]


def _ref(master, rows, B):
    """mk_ref's compositions for the compared rows of a mode on its largest batch"""
    return MK.ref(MK.tenant_of(master)[numpy.arange(B) if rows is None else numpy.asarray(rows)])


def run_modes(eng, keys, modes, sizes_of, what):
    """every mode at every batch of the cell, then its largest batch again with tenant SPOILED's key spoiled (in a
    one-tenant layout, its only tenant's)"""
    for mode in modes:
        dev = mode.upload(eng)
        sizes = sizes_of(mode)
        for b in sizes:
            mode.check(mode.call(eng, dev, (keys, mode.master, None), b), b, what)
        b = sizes[-1]
        counts = MK.truncate(mode.master, b)
        spoiled = SPOILED if len(counts) > SPOILED else 0
        got = mode.call(eng, dev, (keys, mode.master, spoiled), b)
        sel, eq = mode.row_equal(got, b)
        owner = MK.tenant_of(counts)[sel]
        assert eq[owner != spoiled].all(), (what, mode.name, b, 'a tenant without the spoiled key changed')
        mine = eq[owner == spoiled]
        assert mine.size, (what, mode.name, b, 'the spoiled tenant has no rows')
        if mode.key_free:
            assert mine.all(), (what, mode.name, b)
        else:
            assert not mine.all(), (what, mode.name, b, 'the spoiled key gave the right bits')


# ---- bootstrap, n = 25 ----------------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def keys():
    return [O.OracleKeys(20261020 + i) for i in range(KEYS)]


def batches(schedule, pairs=False):
    """ciphertext batches around the wave, or (pairs) odd job batches of extract2 whose 2 B ciphertexts are placed
    around it; the stagger applies to single waves, the chunk schedules to multi-wave launches"""
    w = W()
    if pairs:
        half = w // 2
        sizes = sorted({1, 3, w + 1} | ({half} if half % 2 else {half - 1, half + 1}))
        count = [2 * b for b in sizes]
    else:
        sizes = [1, 2, 3, w - 1, w, w + 1, 2 * w + 3]
        count = sizes
    if schedule == 'stagger0':
        return [b for b, c in zip(sizes, count) if c <= w]
    if schedule in ('one_chunk', 'force4'):
        return [b for b, c in zip(sizes, count) if c > w]
    return sizes


@pytest.fixture(scope='module')
def n25(keys):
    """the modes at n = 25 on each key's first 25 rows, each on the largest batch any cell uses, with layouts cycling
    through LAYOUTS"""
    n, B, J = 25, 2 * W() + 3, W() + 1
    bks = [k.bk[:n] for k in keys]
    t = O.phase_to_t32
    lay = iter(LAYOUTS * 10)
    nxt = lambda M: layout(next(lay), M)                # noqa: E731
    modes = [mk_gate('nand', n, bks, t(1, 8), -1, -1, 2**29, True, 2001, B, nxt(B)),
             mk_gate('xor', n, bks, t(1, 4), 2, 2, -2**31, True, 2002, B, nxt(B)),
             mk_gate('one_input', n, bks, 777777, -1, 9, 123456789, False, 2003, B, nxt(B)),
             mk_x2('mux_jobs', n, bks, (t(-1, 8), 1, 1, True), (t(1, 8) + 4321, -1, 3, True), 2**29, 2004, J, nxt(J)),
             mk_x2('job_b_one_input', n, bks, (t(-1, 8), 1, 1, True), (-55555, 3, 7, False), 123456789, 2005, J,
                   nxt(J))]
    for L in (0, 1, 2):
        for per_ct in (False, True):
            for two in (False, True):
                name = 'lut_L%d_%s_%s' % (L, 'stride1024' if per_ct else 'stride0', 'in2' if two else 'no_in2')
                modes.append(mk_lut(name, n, bks, L, per_ct, two, 2100 + 4 * L + 2 * per_ct + two, B, nxt(B)))
    modes.append(mk_glwe('glwe', n, bks, 2200, B, nxt(B)))
    return bks, modes


def test_layouts_cover_the_matrix(n25):
    """every layout kind occurs, extract2 has a mixed and a one-per-tenant layout; 'mixed' truncated at W - 1, W,
    W + 1 and 2W + 3 has idle tenants first, inside and last, and boundaries at both slot parities"""
    _, modes = n25
    w = W()
    kind = lambda m: 'one' if len(m.master) == 1 else 'ones' if all(c == 1 for c in m.master) else 'mixed'  # noqa
    assert {kind(m) for m in modes if m.kind != 'x2'} == set(LAYOUTS)
    assert {kind(m) for m in modes if m.kind == 'x2'} == {'mixed', 'ones'}
    mixed = layout('mixed', 2 * w + 3)
    for b in (w - 1, w, w + 1, 2 * w + 3):
        c = MK.truncate(mixed, b)
        ends = numpy.cumsum(c)[:-1]
        inner = ends[(ends > 0) & (ends < b)]
        assert c[0] == 0 and c[-1] == 0 and 0 in c[1:-1], b
        assert (inner % 2 == 0).any() and (inner % 2 == 1).any(), b


@pytest.mark.parametrize('shape,schedule', CELLS, ids=['%s-%s' % c for c in CELLS])
def test_bootstrap_n25(monkeypatch, n25, shape, schedule):
    """n = 25: every mode at every batch of the cell, every output row compared"""
    bks, modes = n25
    eng = engine(monkeypatch, shape, schedule)
    keys = Keys(eng, bks)
    run_modes(eng, keys, modes, lambda mode: batches(schedule, pairs=mode.kind == 'x2'),
              '%s/%s n=25' % (shape, schedule))


# ---- bootstrap, n = 500 ---------------------------------------------------------------------------------------------

N500_FULL = (1, 5, 37)


def sample_rows(B):
    """16 rows of a large batch: the first two, the last three (the last full 2-ciphertext CTA and the odd one) and
    random ones"""
    rows = {0, 1, B - 3, B - 2, B - 1}
    rng = G.rs(B)
    while len(rows) < 16:
        rows.add(int(rng.randint(0, B)))
    return sorted(rows)


@pytest.fixture(scope='module')
def n500(keys):
    """NAND on real encryptions under each row's tenant key, extract2, LUT at L = 2 with per-ciphertext test vectors
    and a second input, GLWE; the oracle on every row of the small batches and on sampled rows of 2W + 3"""
    n, B = 500, 2 * W() + 3
    master = layout('mixed', B)
    rows = numpy.array(sorted(set(range(N500_FULL[-1])) | set(sample_rows(B))))
    bks = [k.bk for k in keys]
    rng = G.rs(2300)
    bits = rng.randint(0, 2, (2, B)).astype(bool)
    key_row = MK.tenant_of(master) % KEYS
    x = [(numpy.empty((B, n), numpy.int32), numpy.empty(B, numpy.int32)) for _ in range(2)]
    for k in range(KEYS):
        idx = numpy.flatnonzero(key_row == k)
        for i in range(2):
            a, b = keys[k].encrypt(bits[i][idx])
            x[i][0][idx], x[i][1][idx] = a, b
    num, den, sa, sb = O.GATE_TABLE['nand']
    nand = mk_gate('nand', n, bks, O.phase_to_t32(num, den), sa, sb, int(O.MU), True, 0, B, master, rows, x=tuple(x))
    nand.truth = ~(bits[0] & bits[1])
    t = O.phase_to_t32
    return [nand,
            mk_x2('mux_jobs', n, bks, (t(-1, 8), 1, 1, True), (t(1, 8) + 4321, -1, 3, True), 2**29, 2301, B, master,
                  rows),
            mk_lut('lut_L2', n, bks, 2, True, True, 2302, B, master, rows),
            mk_glwe('glwe', n, bks, 2303, B, master, rows)]


def mk_keyswitch_ptrs(ks_dev, tenants, key_of=lambda t: t % KEYS):
    return [host(ctypes.c_void_p, [ks_dev[key_of(t)][i].data_ptr() for t in range(tenants)]) for i in range(3)]


def test_bootstrap_n500(monkeypatch, keys, n500):
    """n = 500 at B = 1, 5, 37 (every row) and 2W + 3 (sampled rows); the NAND outputs, key-switched by nb_mk_keyswitch
    with each tenant's key, decrypt under each tenant's key to the truth table at every batch"""
    eng = engine(monkeypatch)
    bk_keys = Keys(eng, [k.bk for k in keys])
    sizes = list(N500_FULL) + [2 * W() + 3]
    nand_out = {}
    for mode in n500:
        dev = mode.upload(eng)
        for b in sizes:
            got = mode.call(eng, dev, (bk_keys, mode.master, None), b)
            mode.check(got, b, 'n=500')
            if mode is n500[0]:
                nand_out[b] = got
    ks = [tuple(eng.to_device(x) for x in k.ks) for k in keys]
    nand = n500[0]
    for b in sizes:
        ext_a, ext_b = (eng.to_device(x) for x in nand_out[b])       # alive until the key switch has run
        counts = MK.truncate(nand.master, b)
        ra, rb = eng.empty((b, 500), torch.int32), eng.empty((b,), torch.int32)
        eng._call('nb_mk_keyswitch', ext_a.data_ptr(), ext_b.data_ptr(), None, None, 0,
                  *mk_keyswitch_ptrs(ks, len(counts)), sizes_t(counts), len(counts), 1024, 500, 8, 2, ra.data_ptr(),
                  rb.data_ptr(), None, b)
        got = (eng.to_host(ra), eng.to_host(rb))
        key_row = MK.tenant_of(counts) % KEYS
        for k in range(KEYS):
            idx = numpy.flatnonzero(key_row == k)
            assert (keys[k].decrypt((got[0][idx], got[1][idx])) == nand.truth[idx]).all(), (b, k)


# ---- bootstrap, n = 1024 and n = 1 ----------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def dims(keys):
    rng = G.rs(2400)
    big = [O.bk_transform(G.torus32(rng, (1024, 2, 2, 2, N))) for _ in range(KEYS)]
    small = [k.bk[:1] for k in keys]
    t = O.phase_to_t32
    ones = [1, 1, 1]
    return [(big, [mk_gate('nand', 1024, big, t(1, 8), -1, -1, 2**29, True, 2401, 3, ones),
                   mk_lut('lut_L2', 1024, big, 2, True, True, 2402, 3, ones),
                   mk_glwe('glwe', 1024, big, 2403, 3, ones)]),
            (small, [mk_gate('nand', 1, small, t(1, 8), -1, -1, 2**29, True, 2404, 3, ones),
                     mk_x2('mux_jobs', 1, small, (t(-1, 8), 1, 1, True), (t(1, 8) + 4321, -1, 3, True), 2**29, 2405,
                           3, ones),
                     mk_glwe('glwe', 1, small, 2406, 3, ones)])]


def test_bootstrap_dimensions(monkeypatch, dims):
    """n = 1024 (LWE_N_MAX) on a random integral key per tenant, and n = 1 on each oracle key's first row: B = 3 as
    (1, 1, 1), with the spoiled-key repeat"""
    eng = engine(monkeypatch)
    for bks, modes in dims:
        keys = Keys(eng, bks)
        run_modes(eng, keys, modes, lambda mode: [3], 'n=%d' % modes[0].n)
        del keys


# ---- nb_mk_keyswitch ------------------------------------------------------------------------------------------------

KS_MMA_MIN = 64
KS_GUARD = 256                              # guard rows: more than the padding of a GEMM tile
POISON_ROWS = 3
REGISTERED = 1                              # the key (and so the tenants t % 3 == 1) whose planes are registered


@pytest.fixture(scope='module')
def ks_env(keys):
    """one engine with NUFHE_B200_KS_MMA_MIN = KS_MMA_MIN; the three oracle keys and two edge keys on the device, the
    planes of key REGISTERED registered"""
    mp = pytest.MonkeyPatch()
    try:
        eng = engine(mp, extra={'NUFHE_B200_KS_MMA_MIN': str(KS_MMA_MIN)})
    finally:
        mp.undo()
    hosts = [k.ks for k in keys] + [K.edge_key('tagged', G.rs(2500)), K.edge_key('min_word', G.rs(2501))]
    dev = [tuple(eng.to_device(x) for x in h) for h in hosts]
    planes = eng.ks_prepare(dev[REGISTERED][0], dev[REGISTERED][1])
    assert planes is not None
    return eng, hosts, dev, planes


def ks_case(env, counts, seed, key_of=lambda t: t % KEYS):
    """inputs of one mix: edge rows first (ks_ref.edge_rows), fold pairs that add up to them, the oracle per tenant"""
    eng, hosts, dev, planes = env
    B = sum(counts)
    rng = G.rs(seed)
    a = K.edge_rows(rng, B)
    b = G.torus32(rng, (B,))
    a1, a2 = K.fold_pair(rng, a)
    b1 = G.torus32(rng, (B,))
    c = 2**29
    b2 = K.i32(K.u32(b) - K.u32(b1) - c)
    owner = MK.tenant_of(counts)
    want_a, want_b = numpy.empty((B, 500), numpy.int32), numpy.empty(B, numpy.int32)
    want_cv = numpy.empty(B, numpy.float32)
    keys_used = numpy.array([key_of(t) for t in range(len(counts))], int)[owner] if B else numpy.zeros(0, int)
    for k in numpy.unique(keys_used):
        idx = numpy.flatnonzero(keys_used == k)
        wa, wb, _ = O.lwe_keyswitch(*hosts[k], a[idx], b[idx])
        want_a[idx], want_b[idx] = wa, wb
        want_cv[idx] = K.variance(hosts[k][2], a[idx])
    return dict(counts=counts, key_of=key_of, plain=((a, b), None, 0), fold=((a1, b1), (a2, b2), c),
                want=(want_a, want_b, want_cv))


def _poisoned(eng, x, poison):
    x = numpy.asarray(x, numpy.int32)
    tail = numpy.full((POISON_ROWS,) + x.shape[1:], poison, numpy.int32)
    return eng.to_device(numpy.concatenate([x, tail]))


def ks_run(env, case, fold, with_cv):
    """nb_mk_keyswitch of one mix: (res_a, res_b, res_cv as uint32 or None); the guards must be intact"""
    eng, hosts, dev, planes = env
    counts, key_of = case['counts'], case['key_of']
    B, T = sum(counts), len(counts)
    src1, src2, c = case['fold'] if fold else case['plain']
    keep = []

    def src(x):
        if x is None:
            return None, None
        pa, pb = _poisoned(eng, x[0], int(K.i32(K.ALL_THREE))), _poisoned(eng, x[1], 2**31 - 1)
        keep.extend((pa, pb))
        return pa.data_ptr(), pb.data_ptr()
    s1a, s1b = src(src1)
    s2a, s2b = src(src2)
    ra = torch.full((B + 2 * KS_GUARD, 500), F.SENTINEL, dtype=torch.int32, device=eng.device)
    rb = torch.full((B + 2 * KS_GUARD,), F.SENTINEL, dtype=torch.int32, device=eng.device)
    rcv = torch.full((B + 2 * KS_GUARD,), F.SENTINEL, dtype=torch.int32, device=eng.device)
    eng._call('nb_mk_keyswitch', s1a, s1b, s2a, s2b, c, *mk_keyswitch_ptrs(dev, T, key_of), sizes_t(counts), T, 1024,
              500, 8, 2, ra[KS_GUARD].data_ptr(), rb[KS_GUARD].data_ptr(),
              rcv[KS_GUARD].data_ptr() if with_cv else None, B)
    out = []
    for buf, what in ((ra, 'res_a'), (rb, 'res_b'), (rcv, 'res_cv')):
        h = buf.cpu().numpy()
        assert (h[:KS_GUARD] == F.SENTINEL).all() and (h[KS_GUARD + B:] == F.SENTINEL).all(), \
            'a store outside the rows of ' + what
        out.append(h[KS_GUARD:KS_GUARD + B])
    if not with_cv:
        assert (out[2] == F.SENTINEL).all(), 'res_cv = NULL, yet variances were stored'
    return out[0], out[1], out[2].view(numpy.uint32) if with_cv else None


def ks_failures(env, case, what):
    """every row of all four calls (plain / fold, with / without res_cv) against the oracle and the fixed-shape
    variance"""
    wa, wb, wcv = case['want']
    out = []
    for fold in (False, True):
        for with_cv in (True, False):
            a, b, cv = ks_run(env, case, fold, with_cv)
            tag = '%s%s%s' % (what, ' fold' if fold else '', '' if with_cv else ' no-cv')
            bad = numpy.flatnonzero((a != wa).any(axis=1) | (b != wb))
            if bad.size:
                out.append('%s: %d rows differ from the oracle (first %s)' % (tag, bad.size, bad[:4].tolist()))
            if cv is not None:
                cv_bad = numpy.flatnonzero(cv != wcv.view(numpy.uint32))
                if cv_bad.size:
                    out.append('%s: %d variances differ (first %s)' % (tag, cv_bad.size, cv_bad[:4].tolist()))
    return out


def test_keyswitch_split_bands(ks_env):
    """gather-only mixes whose tile count is at both edges of every split band the card reaches"""
    sm = sm_count()
    failures, reached = [], set()
    for i, (s, counts) in enumerate(MK.ks_band_mixes(sm)):
        tiles = MK.ks_tiles(counts, {REGISTERED}, KS_MMA_MIN)
        assert not MK.ks_gemm_tenants(counts, {REGISTERED}, KS_MMA_MIN)
        assert MK.ks_splits(len(tiles), sm) == s
        reached.add(s)
        failures += ks_failures(ks_env, ks_case(ks_env, counts, 2600 + i),
                                'tiles %d (split %d, %d tenants)' % (len(tiles), s, len(counts)))
    assert reached == set(MK.ks_split_bands(sm))
    assert not failures, '\n'.join(failures)


@pytest.mark.parametrize('split_one', [False, True], ids=['split_gt1', 'split1'])
def test_keyswitch_gemm_beside_gather(ks_env, split_one):
    """a registered tenant at KS_MMA_MIN - 1 rows (gather) and at KS_MMA_MIN (GEMM) beside gather tenants of 31, 32
    and 33 rows, and an edge-key tenant; the GEMM tenant must run the GEMM (zeroed planes change its bits)"""
    eng, hosts, dev, planes = ks_env
    sm = sm_count()
    failures = []
    for j, R in enumerate((KS_MMA_MIN - 1, KS_MMA_MIN)):
        counts = [31, R, 32, 33]                 # tenant 1: key REGISTERED
        if split_one:                            # single-row gather tenants until the SMs are covered without a split
            counts += [1] * max(0, sm // 2 + 1 - len(MK.ks_tiles(counts, {REGISTERED}, KS_MMA_MIN)))
        gemm = MK.ks_gemm_tenants(counts, {REGISTERED}, KS_MMA_MIN)
        assert gemm == ([1] if R >= KS_MMA_MIN else []), gemm
        tiles = MK.ks_tiles(counts, {REGISTERED}, KS_MMA_MIN)
        assert (MK.ks_splits(len(tiles), sm) == 1) == split_one, len(tiles)
        # tenant 3 switches with the tagged edge key
        key_of = lambda t: 3 if t == 3 else t % KEYS            # noqa: E731
        case = ks_case(ks_env, counts, 2700 + 10 * j + split_one, key_of)
        failures += ks_failures(ks_env, case, 'R=%d tiles %d split %d' % (R, len(tiles), MK.ks_splits(len(tiles), sm)))
        if gemm:
            a, _, _ = ks_run(ks_env, case, False, True)
            saved = planes.clone()
            planes.zero_()
            try:
                z, _, _ = ks_run(ks_env, case, False, True)
            finally:
                planes.copy_(saved)
            lo = counts[0]
            assert not (z[lo:lo + R] == a[lo:lo + R]).all(), 'the GEMM tenant did not run on the GEMM'
            assert (numpy.delete(z, numpy.s_[lo:lo + R], 0) == numpy.delete(a, numpy.s_[lo:lo + R], 0)).all()
    assert not failures, '\n'.join(failures)


def test_keyswitch_segments_and_edge_keys(ks_env):
    """segments of 31, 32 and 33 rows in every order, and a mix in which two tenants switch with edge keys (tagged:
    each word encodes its position; every word -2^31)"""
    failures = []
    for i, counts in enumerate(([31, 32, 33], [33, 31, 32], [32, 33, 31, 1, 0, 33])):
        failures += ks_failures(ks_env, ks_case(ks_env, counts, 2800 + i), 'segments %s' % (counts,))
    key_of = lambda t: {1: 3, 2: 4}.get(t, t % KEYS)                # noqa: E731
    failures += ks_failures(ks_env, ks_case(ks_env, [33, 31, 32, 5], 2810, key_of), 'edge keys')
    assert not failures, '\n'.join(failures)


# ---- nb_mk_tree_keyswitch -------------------------------------------------------------------------------------------

TREE_COUNTS = {'255_256_257': (255, 256, 257), '0_1_513': (0, 1, 513), '700x1': (1,) * 700}


def _rand(rng, shape):
    return rng.randint(-2**31, 2**31, size=shape, dtype=numpy.int64).astype(numpy.int32)


def tree_check(eng, a, hosts, counts, key_of, k):
    """nb_mk_tree_keyswitch with each tenant's planes against tree_ref.keyswitch on that tenant's key"""
    R, n = a.shape
    planes = [eng.tree_prepare(eng.to_device(m), eng.to_device(b)) for m, b in hosts]
    out = torch.full((R + 2 * F.GUARD, k + 1, N), F.SENTINEL, dtype=torch.int32, device=eng.device)
    da = eng.to_device(a)                       # alive until the launch has run
    eng._call('nb_mk_tree_keyswitch', da.data_ptr(),
              host(ctypes.c_void_p, [planes[key_of(t)].data_ptr() for t in range(len(counts))]), sizes_t(counts),
              len(counts), n, k, out[F.GUARD].data_ptr(), R)
    got = F.unguard(out, 'out')
    keys_used = numpy.array([key_of(t) for t in range(len(counts))])[MK.tenant_of(counts)]
    for key in numpy.unique(keys_used):
        idx = numpy.flatnonzero(keys_used == key)
        assert (got[idx] == tree_ref.keyswitch(a[idx], *hosts[key])).all(), (counts[:4], key)


@pytest.mark.parametrize('counts', list(TREE_COUNTS), ids=list(TREE_COUNTS))
@pytest.mark.parametrize('n', [500, 25, 1])
@pytest.mark.parametrize('k', [1, 2])
def test_tree_keyswitch(monkeypatch, counts, n, k):
    eng = engine(monkeypatch)
    counts = list(TREE_COUNTS[counts])
    rng = G.rs(2900 + 7 * n + k)
    hosts = [(_rand(rng, (n, 2, k, N)), _rand(rng, (n, 2, N))) for _ in range(KEYS)]
    tree_check(eng, _rand(rng, (sum(counts), n)), hosts, counts, lambda t: t % KEYS, k)


def test_tree_keyswitch_at_the_exactness_bound(monkeypatch):
    """tenant 1 at the exactness bound (every digit -128, key words -2^31 and 2^31 - 1) between random tenants"""
    eng = engine(monkeypatch)
    n, k = 500, 1
    rng = G.rs(2950)
    masks = numpy.full((n, 2, k, N), -2**31, numpy.int32)
    body = numpy.full((n, 2, N), -2**31, numpy.int32)
    masks[:, :, :, 1::2] = 2**31 - 1
    body[:, :, ::3] = 1
    hosts = [(_rand(rng, (n, 2, k, N)), _rand(rng, (n, 2, N))), (masks, body),
             (_rand(rng, (n, 2, k, N)), _rand(rng, (n, 2, N)))]
    counts = [255, 257, 33]
    a = _rand(rng, (sum(counts), n))
    a[255:512] = numpy.int64(0x7f7f8000).astype(numpy.int32)
    tree_check(eng, a, hosts, counts, lambda t: t, k)


# ---- nb_mk_ntt_mac --------------------------------------------------------------------------------------------------

def _field(rng, shape):
    """plain-form field elements with p - 1, 0 and 1 at the first positions"""
    x = rng.randint(0, 2**63, size=shape, dtype=numpy.int64).view(numpy.uint64) % numpy.uint64(O.P)
    flat = x.reshape(-1)
    flat[:64:3], flat[1:64:3], flat[2:64:3] = numpy.uint64(O.P - 1), 0, 1
    flat[-16:] = numpy.uint64(O.P - 1)
    return x


def mac_ref(x, key):
    """out (G, U, N) = sum_r x[:, r] key[r] mod P in Python integers"""
    acc = numpy.zeros((x.shape[0], key.shape[1], N), object)
    for r in range(x.shape[1]):
        acc = acc + x[:, r, None, :].astype(object) * key[None, r].astype(object)
    return (acc % O.P).astype(numpy.uint64)


@pytest.mark.parametrize('groups', [(0, 1, 2, 0, 3), (1,) * 300], ids=['0_1_2_0_3', '300x1'])
def test_ntt_mac(monkeypatch, groups):
    eng = engine(monkeypatch)
    rng = G.rs(3000 + len(groups))
    R, U = 4, 3                                 # U = 3: two output tiles of 2
    Gs = sum(groups)
    keys = [_field(rng, (R, U, N)) for _ in range(KEYS)]
    x = _field(rng, (Gs, R, N))
    out = torch.full((Gs + 2 * F.GUARD, U, N), -1, dtype=torch.int64, device=eng.device)
    dkeys = [eng.to_device(k) for k in keys]
    dx = eng.to_device(x)                       # alive until the launch has run
    eng._call('nb_mk_ntt_mac', dx.data_ptr(),
              host(ctypes.c_void_p, [dkeys[t % KEYS].data_ptr() for t in range(len(groups))]), sizes_t(groups),
              len(groups), out[F.GUARD].data_ptr(), R, U, Gs)
    h = out.cpu().numpy()
    assert (h[:F.GUARD] == -1).all() and (h[-F.GUARD:] == -1).all(), 'a store outside the groups'
    got = h[F.GUARD:-F.GUARD].view(numpy.uint64)
    owner = MK.group_tenants(groups) % KEYS
    for k in range(KEYS):
        idx = numpy.flatnonzero(owner == k)
        if idx.size:
            assert (got[idx] == mac_ref(x[idx], keys[k])).all(), (groups[:5], k)
