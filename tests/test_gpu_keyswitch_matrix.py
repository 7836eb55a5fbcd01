"""Every code path of nb_keyswitch in every launch shape the card reaches, against the exact CPU oracle on every row.

nb_keyswitch picks one of three kernels (capi.cu): keyswitch_mma_kernel (a registered key, batch >= the engine's
threshold, aligned pointers) with K split 1 to 8 ways, keyswitch_kernel (the scheme's parameters) with 1 to 128 slices of
j and ks_cv_finalize_kernel, and keyswitch_generic_kernel (any other decomposition).  tests/ks_ref.py restates the
dispatch rules; the batches here sit at both edges of every split band of both fast paths on this card's SM count.
K split 16 needs 256 SMs, so no H100 reaches it.

Two engines share the device: one with NUFHE_B200_KS_MMA_MIN=1 and a prepared key (every batch on the GEMM), one with a
threshold no batch reaches (every batch on the gather kernel).  Every call goes through the C ABI with its outputs inside
sentinel-filled buffers, guard words before and after, and source rows past the batch poisoned.  Every cell requires
res_a and res_b equal to O.lwe_keyswitch on all rows, intact guards, and variances equal bit for bit to the fixed-shape
float32 sum (ks_ref.variance) -- for the generic kernel, to the oracle's running sum, which adds in the same order."""
import contextlib
import ctypes
import gc
import os

import numpy
import pytest
import torch

import gen_inputs as G
import ks_ref as K
from nufhe_b200 import _native
from oracle import oracle as O

pytestmark = pytest.mark.gpu

SENTINEL = 0x5A5A5A5A
# sentinel words before and after every output: more than the 255 padded rows of a GEMM tile, so that a store into the
# padding of the last tile lands in the guard rather than in another allocation
GUARD_WORDS = 256 * 512
POISON_ROWS = 3             # source rows past the batch: all digits 3, b = 2^31 - 1
MUX_C = 2**29               # gate_mux's (0, 1/8)


def _engine(threshold):
    from nufhe_b200.engine import Engine
    old = os.environ.get('NUFHE_B200_KS_MMA_MIN')
    os.environ['NUFHE_B200_KS_MMA_MIN'] = str(threshold)
    try:
        return Engine()
    finally:
        if old is None:
            del os.environ['NUFHE_B200_KS_MMA_MIN']
        else:
            os.environ['NUFHE_B200_KS_MMA_MIN'] = old


@pytest.fixture(scope='module')
def engs():
    """(GEMM engine, gather engine)"""
    return _engine(1), _engine(1 << 62)


@pytest.fixture(scope='module')
def sm_count():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


@pytest.fixture(scope='module')
def generated():
    return O.OracleKeys(G.GATE_SEED).ks


class Guarded:
    """`count` int32 words of output, `shift` words past GUARD_WORDS sentinel words, and GUARD_WORDS after them"""

    def __init__(self, eng, count, shift=0):
        self.start, self.count = GUARD_WORDS + shift, count
        self.buf = torch.full((count + 2 * GUARD_WORDS + shift,), SENTINEL, dtype=torch.int32, device=eng.device)
        self.ptr = self.buf.data_ptr() + 4 * self.start

    def read(self):
        """(body as int32, guards intact)"""
        h = self.buf.cpu().numpy()
        intact = (h[:self.start] == SENTINEL).all() and (h[self.start + self.count:] == SENTINEL).all()
        return h[self.start:self.start + self.count], bool(intact)


def _source(eng, rows, poison, shift=0):
    """rows then POISON_ROWS rows of `poison` on the device, starting `shift` words into the buffer: (tensor, pointer)"""
    rows = numpy.asarray(rows, numpy.int32)
    width = rows[0].size if rows.ndim > 1 else 1
    flat = numpy.full(shift + rows.size + POISON_ROWS * width, poison, numpy.int32)
    flat[shift:shift + rows.size] = rows.ravel()
    t = eng.to_device(flat)
    return t, t.data_ptr() + 4 * shift


def fold(src1, src2, c):
    """(a, b) of src1 + src2 + (0, c) mod 2^32, as nb_keyswitch forms it"""
    if src2 is None:
        return src1[0], K.i32(K.u32(src1[1]) + c)
    return K.i32(K.u32(src1[0]) + K.u32(src2[0])), K.i32(K.u32(src1[1]) + K.u32(src2[1]) + c)


def run(eng, ks, src1, src2=None, c=0, src_shift=(0, 0), res_shift=0):
    """nb_keyswitch(ks on the device, host sources) through the C ABI: (res_a, res_b, res_cv as uint32, guards intact)"""
    in_size, t, base, n = ks[0].shape
    B = src1[1].size
    keep = []

    def source(x, shift):
        if x is None:
            return None, None
        a, pa = _source(eng, x[0], int(K.i32(K.ALL_THREE)), shift)
        b, pb = _source(eng, x[1], 2**31 - 1)
        keep.extend((a, b))
        return pa, pb

    s1a, s1b = source(src1, src_shift[0])
    s2a, s2b = source(src2, src_shift[1])
    ra, rb, rcv = Guarded(eng, B * n, res_shift), Guarded(eng, B), Guarded(eng, B)
    eng._call('nb_keyswitch', s1a, s1b, s2a, s2b, int(K.i32(c)), ks[0].data_ptr(), ks[1].data_ptr(),
              ks[2].data_ptr(), in_size, n, t, int(base).bit_length() - 1, ra.ptr, rb.ptr, rcv.ptr, B)
    (a, ga), (b, gb), (cv, gc_) = ra.read(), rb.read(), rcv.read()
    return a.reshape(B, n), b, cv.view(numpy.uint32), ga and gb and gc_


def check(what, got, want, cv_want):
    """failures of one cell: rows of a or b off the oracle, broken guards, variance bits off `cv_want`"""
    a, b, cv, intact = got
    wa, wb = want
    bad = numpy.flatnonzero((a != wa).any(axis=1) | (b != wb))
    out = []
    if bad.size:
        out.append('%s: %d rows differ from the oracle (first %s)' % (what, bad.size, bad[:4].tolist()))
    if not intact:
        out.append('%s: a store outside the batch' % what)
    cv_bad = numpy.flatnonzero(cv != numpy.asarray(cv_want, numpy.float32).view(numpy.uint32))
    if cv_bad.size:
        out.append('%s: %d variances differ (first %s)' % (what, cv_bad.size, cv_bad[:4].tolist()))
    return out


@contextlib.contextmanager
def zeroed(planes):
    """the planes zeroed for the block: a GEMM launch with the key then gives other bits"""
    saved = planes.clone()
    planes.zero_()
    try:
        yield
    finally:
        planes.copy_(saved)


def same(x, y):
    return all((u == v).all() for u, v in zip(x[:3], y[:3]))


class Paths:
    """a host key on both engines; the GEMM engine's copy prepared"""

    def __init__(self, engs, host, expect_registered=True):
        self.host = host
        self.gemm = tuple(engs[0].to_device(x) for x in host)
        self.gather = tuple(engs[1].to_device(x) for x in host)
        self.planes = engs[0].ks_prepare(self.gemm[0], self.gemm[1])
        assert (self.planes is not None) == expect_registered

    def cells(self, engs, what, src1, src2=None, c=0):
        """both paths of one cell against the oracle and the fixed-shape variance; identical variance bits"""
        sa, sb = fold(src1, src2, c)
        want = O.lwe_keyswitch(*self.host, sa, sb)[:2]
        cv_want = K.variance(self.host[2], sa)
        x = run(engs[0], self.gemm, src1, src2, c)
        y = run(engs[1], self.gather, src1, src2, c)
        out = check(what + ' gemm', x, want, cv_want) + check(what + ' gather', y, want, cv_want)
        if not (x[2] == y[2]).all():
            out.append(what + ': the two paths give different variance bits')
        return out


def _inputs(rng, B, with_fold):
    """edge rows (ks_ref.edge_rows); with the fold, pairs that wrap to them, and c = 1/8"""
    a = K.edge_rows(rng, B)
    b = G.torus32(rng, (B,))
    if not with_fold:
        return (a, b), None, 0
    a1, a2 = K.fold_pair(rng, a)
    return (a1, b), (a2, G.torus32(rng, (B,))), MUX_C


def _shape(B, sm):
    return 'B=%d (gather splits %d, j_per %d; gemm splits %d)' % (
        B, K.gather_launch(B, sm)[2], K.gather_launch(B, sm)[3], K.mma_launch(B, sm)[2])


def test_launch_shapes(engs, sm_count, generated):
    """the generated key at both edges of every split band of both fast paths, 1, 256 and multi-wave batches; every
    other cell folds src2 + (0, c) as gate_mux does"""
    paths = Paths(engs, generated)
    rng = G.rs(900)
    failures = []
    batches = K.matrix_batches(sm_count)
    for i, B in enumerate(batches):
        src1, src2, c = _inputs(rng, B, i % 2 == 1)
        failures += paths.cells(engs, _shape(B, sm_count) + (' fold' if src2 else ''), src1, src2, c)
    # every split value of both paths was reached
    assert {K.gather_launch(B, sm_count)[2] for B in batches} == set(K.gather_bands(sm_count))
    assert {K.mma_launch(B, sm_count)[2] for B in batches} == set(K.mma_bands(sm_count))
    assert not failures, '\n'.join(failures)
    # and the GEMM engine ran the GEMM: without its planes the bits change
    src1, _, _ = _inputs(rng, 1, False)
    x = run(engs[0], paths.gemm, src1)
    with zeroed(paths.planes):
        assert not same(run(engs[0], paths.gemm, src1), x)


@pytest.mark.parametrize('kind', K.KEY_KINDS)
def test_key_edges(engs, sm_count, generated, kind):
    """edge keys: random, every byte 0xFF, every word -2^31, and tagged (each word encodes its (j, k, d, x)), at one
    batch in each GEMM split band and the gather kernel's 128-, 13-, 6- and 1-way splits"""
    host = generated if kind == 'generated' else K.edge_key(kind, G.rs(910))
    paths = Paths(engs, host)
    rng = G.rs(911)
    failures = []
    for i, B in enumerate((1, 300, 600, 4097)):
        src1, src2, c = _inputs(rng, B, i % 2 == 0)
        failures += paths.cells(engs, '%s %s%s' % (kind, _shape(B, sm_count), ' fold' if src2 else ''), src1, src2, c)
    assert not failures, '\n'.join(failures)


def test_padded_key_stays_on_the_gather_kernel(engs, sm_count):
    """a key whose d = 0 rows are not zero is not registered; the GEMM, which drops those rows, would give other bits"""
    paths = Paths(engs, K.edge_key('pad', G.rs(920)), expect_registered=False)
    rng = G.rs(921)
    failures = []
    for i, B in enumerate(sorted({b for bs in K.mma_batches(sm_count).values() for b in bs} | set(K.MULTI_WAVE))):
        src1, src2, c = _inputs(rng, B, i % 2 == 0)
        failures += paths.cells(engs, 'pad ' + _shape(B, sm_count), src1, src2, c)
    assert not failures, '\n'.join(failures)


@pytest.mark.parametrize('where', ['src1_a', 'src2_a', 'res_a'])
def test_misaligned_pointers_take_the_gather_kernel(engs, generated, where):
    """src_a 4 bytes past 16-byte alignment, or res_a 4 bytes past 8-byte alignment: the gather kernel runs (zeroed
    planes change nothing), with the oracle's bits and intact guards"""
    paths = Paths(engs, generated)
    eng = engs[0]
    rng = G.rs(930)
    B = 300
    src1, src2, c = _inputs(rng, B, True)
    sa, sb = fold(src1, src2, c)
    want = O.lwe_keyswitch(*generated, sa, sb)[:2]
    cv_want = K.variance(generated[2], sa)
    kw = dict(src_shift=(int(where == 'src1_a'), int(where == 'src2_a')), res_shift=int(where == 'res_a'))
    got = run(eng, paths.gemm, src1, src2, c, **kw)
    assert not check(where, got, want, cv_want)
    with zeroed(paths.planes):
        assert same(run(eng, paths.gemm, src1, src2, c, **kw), got)
        assert not same(run(eng, paths.gemm, src1, src2, c), got)      # aligned: the GEMM, which reads the planes


GENERIC = [(8, 2, 2048, 500), (4, 4, 1024, 500)] + [(t, lb, 16, n) for t, lb in ((3, 10), (31, 1)) for n in (1, 7, 511)]


@pytest.mark.parametrize('t,log2_base,in_size,n', GENERIC)
def test_generic_kernel(engs, t, log2_base, in_size, n):
    """keyswitch_generic_kernel at the edges of the C ABI (t * log2_base <= 31, n <= 511), batches 1, 7 and 513 with
    and without the fold: every row equals the oracle, variances equal its running float32 sum bit for bit"""
    eng = engs[1]
    rng = G.rs(940 + t * 100 + n)
    base = 1 << log2_base
    host = (G.torus32(rng, (in_size, t, base, n)), G.torus32(rng, (in_size, t, base)),
            rng.uniform(0.0, 1e-6, size=(in_size, t, base)).astype(numpy.float32))
    ks = tuple(eng.to_device(x) for x in host)
    failures = []
    for B in (1, 7, 513):
        for with_fold in (False, True):
            a = G.torus32(rng, (B, in_size))
            a[0] = -1
            if B > 1:
                a[1] = -2**31
            src1 = (a, G.torus32(rng, (B,)))
            src2, c = (None, 0)
            if with_fold:
                a1, a2 = K.fold_pair(rng, a)
                src1, src2, c = (a1, src1[1]), (a2, G.torus32(rng, (B,))), MUX_C
            sa, sb = fold(src1, src2, c)
            wa, wb, wcv = O.lwe_keyswitch(*host, sa, sb)
            failures += check('B=%d fold=%s' % (B, with_fold), run(eng, ks, src1, src2, c), (wa, wb), wcv)
    assert not failures, '\n'.join(failures)


def test_refusals(engs):
    """n = 512 is unsupported; t * log2_base = 32, t = 0 and log2_base = 0 are invalid; batch 0 is a no-op.  None of
    them writes to the outputs"""
    eng = engs[1]
    host = (numpy.zeros((16, 4, 2, 7), numpy.int32), numpy.zeros((16, 4, 2), numpy.int32),
            numpy.zeros((16, 4, 2), numpy.float32))
    ks = tuple(eng.to_device(x) for x in host)
    src_a, pa = _source(eng, numpy.ones((2, 16), numpy.int32), 0)
    src_b, pb = _source(eng, numpy.ones(2, numpy.int32), 0)
    outs = Guarded(eng, 2 * 512), Guarded(eng, 2), Guarded(eng, 2)
    torch.cuda.synchronize()

    def call(n, t, log2_base, batch):
        return eng.lib.nb_keyswitch(eng.handle, pa, pb, None, None, 0, ks[0].data_ptr(), ks[1].data_ptr(),
                                    ks[2].data_ptr(), 16, n, t, log2_base, outs[0].ptr, outs[1].ptr, outs[2].ptr,
                                    batch)
    assert call(512, 4, 1, 2) == _native.NB_EUNSUPPORTED
    for t, lb in ((32, 1), (4, 8), (1, 32), (0, 1), (4, 0)):
        assert call(7, t, lb, 2) == _native.NB_EINVAL, (t, lb)
    assert call(7, 4, 1, 0) == _native.NB_OK
    torch.cuda.synchronize()
    for o in outs:
        body, intact = o.read()
        assert intact and (body == SENTINEL).all()


# ---- registrations (nb_ks_prepare, Engine.ks_prepare) ---------------------------------------------------------------

def _src(seed, B):
    rng = G.rs(seed)
    return (G.torus32(rng, (B, 1024)), G.torus32(rng, (B,)))


def _want(host, src):
    return O.lwe_keyswitch(*host, src[0], src[1])[:2]


def _equal(got, want):
    return (got[0] == want[0]).all() and (got[1] == want[1]).all() and got[3]


def test_two_keys_and_a_prepare_into_the_other_keys_planes(engs, generated):
    """two keys registered on one engine each run on the GEMM; preparing key A into the buffer of B's planes drops B's
    registration (B falls back to the gather kernel) and moves A's to that buffer"""
    eng = engs[0]
    hosts = (generated, K.edge_key('random', G.rs(950)))
    keys = [tuple(eng.to_device(x) for x in h) for h in hosts]
    planes = [eng.ks_prepare(k[0], k[1]) for k in keys]
    assert all(p is not None for p in planes)
    src = _src(951, 300)
    wants = [_want(h, src) for h in hosts]
    for k, p, w in zip(keys, planes, wants):
        got = run(eng, k, src)
        assert _equal(got, w)
        with zeroed(p):
            assert not same(run(eng, k, src), got)
    a, b = keys
    registered = ctypes.c_int(0)
    eng._call('nb_ks_prepare', a[0].data_ptr(), a[1].data_ptr(), planes[1].data_ptr(), 1024, 500, 8, 2,
              ctypes.addressof(registered))
    try:
        assert registered.value == 1
        got_a, got_b = run(eng, a, src), run(eng, b, src)
        assert _equal(got_a, wants[0]) and _equal(got_b, wants[1])
        with zeroed(planes[1]):
            assert same(run(eng, b, src), got_b)                 # B: the gather kernel
            assert not same(run(eng, a, src), got_a)             # A: the GEMM on the planes it was prepared into
        with zeroed(planes[0]):
            assert same(run(eng, a, src), got_a)
    finally:
        eng.lib.nb_ks_forget(eng.handle, a[0].data_ptr())       # the raw prepare is outside the engine's bookkeeping


def _key_in_one_block(eng, host):
    """ks_a and ks_b as views of one allocation, and ks_cv: a key of the same size allocated after this one is freed
    takes the same block of the caching allocator, so both addresses repeat"""
    ks_a, ks_b, ks_cv = host
    buf = eng.to_device(numpy.concatenate([ks_a.ravel(), ks_b.ravel()]))
    return [buf[:ks_a.size].view(ks_a.shape), buf[ks_a.size:].view(ks_b.shape), eng.to_device(ks_cv)]


def test_freed_key_leaves_no_registration(engs, generated):
    """the key's tensors freed while its planes live: a new key at the same addresses must not be switched with the old
    key's planes"""
    eng = engs[0]
    gc.collect()
    ks = _key_in_one_block(eng, generated)
    planes = eng.ks_prepare(ks[0], ks[1])
    assert planes is not None
    addr = (ks[0].data_ptr(), ks[1].data_ptr())
    del ks
    gc.collect()
    other = K.edge_key('random', G.rs(960))
    ks = _key_in_one_block(eng, other)
    if (ks[0].data_ptr(), ks[1].data_ptr()) != addr:
        pytest.skip('the allocator placed the new key elsewhere, so the case does not arise')
    src = _src(961, 4096)
    assert _equal(run(eng, ks, src), _want(other, src))
    del planes


def test_second_prepare_survives_the_first_planes(engs, generated):
    """the same key prepared into two plane buffers: freeing the first keeps the key registered on the second"""
    eng = engs[0]
    ks = [eng.to_device(x) for x in generated]
    first = eng.ks_prepare(ks[0], ks[1])
    second = eng.ks_prepare(ks[0], ks[1])
    assert first is not None and second is not None
    del first
    gc.collect()
    src = _src(970, 300)
    got = run(eng, ks, src)
    assert _equal(got, _want(generated, src))
    with zeroed(second):
        assert not same(run(eng, ks, src), got), 'the key fell back to the gather kernel'


# ---- the public API ------------------------------------------------------------------------------------------------

def test_vm_gates_on_the_gemm(generated):
    """gate_nand and gate_mux at batch 4096 through a VirtualMachine, whose key switch runs on the GEMM: every row
    equals the oracle's key switch of the fused bootstrap's output, and rows at both ends equal the oracle's whole gate
    (the whole gate on all rows is test_gpu_gates.py's, on the gather kernel)"""
    import nufhe_b200 as nufhe
    from nufhe_b200.lwe import LweSampleArray
    ctx = nufhe.Context(rng=nufhe.DeterministicRNG(G.GATE_SEED))
    _, ck = ctx.make_key_pair()
    vm = ctx.make_virtual_machine(ck)
    eng = ctx.thread
    planes = ck.keyswitch_key._gemm_planes[2]
    assert planes is not None
    ks_dev = ck.keyswitch_key.device_arrays()
    assert all((eng.to_host(d) == h).all() for d, h in zip(ks_dev[:2], generated[:2]))   # the oracle's key
    keys = O.OracleKeys(G.GATE_SEED)
    bk_int = eng.bk_prepare(eng.to_device(keys.bk))
    B = 4096
    rng = G.rs(980)
    bits = [rng.randint(0, 2, B).astype(bool) for _ in range(3)]
    cts = [keys.encrypt(x) for x in bits]
    d = [LweSampleArray(ck.params.in_out_params, eng.to_device(x[0]), eng.to_device(x[1]),
                        torch.zeros(B, dtype=torch.float32, device=eng.device)) for x in cts]
    dev = [(x.a, x.b) for x in d]
    ends = numpy.r_[0:4, B - 4:B]
    sub = lambda x: (x[0][ends], x[1][ends])      # noqa: E731

    r = vm.gate_nand(d[0], d[1])
    got = (eng.to_host(r.a), eng.to_host(r.b))
    num, den, sa, sb = O.GATE_TABLE['nand']
    ext = eng.bootstrap_extract(dev[0], dev[1], O.phase_to_t32(num, den), sa, sb, O.MU, bk_int)
    want = O.lwe_keyswitch(*generated, eng.to_host(ext[0]), eng.to_host(ext[1]))
    assert (got[0] == want[0]).all() and (got[1] == want[1]).all()
    w = O.gate_binary('nand', sub(cts[0]), sub(cts[1]), keys.bk, keys.ks)
    assert (got[0][ends] == w[0]).all() and (got[1][ends] == w[1]).all()
    assert (keys.decrypt(got) == ~(bits[0] & bits[1])).all()
    with zeroed(planes):
        spoiled = vm.gate_nand(d[0], d[1])
        assert not (eng.to_host(spoiled.a) == got[0]).all()

    m = vm.gate_mux(d[0], d[1], d[2])
    got = (eng.to_host(m.a), eng.to_host(m.b))
    and_const = O.phase_to_t32(-1, 8)
    u1, u2 = eng.bootstrap_extract2((dev[0], dev[1], and_const, 1, 1), (dev[0], dev[2], and_const, -1, 1), O.MU, bk_int)
    sa, sb = fold((eng.to_host(u1[0]), eng.to_host(u1[1])), (eng.to_host(u2[0]), eng.to_host(u2[1])),
                  int(O.phase_to_t32(1, 8)))
    want = O.lwe_keyswitch(*generated, sa, sb)
    assert (got[0] == want[0]).all() and (got[1] == want[1]).all()
    w = O.gate_mux(sub(cts[0]), sub(cts[1]), sub(cts[2]), keys.bk, keys.ks)
    assert (got[0][ends] == w[0]).all() and (got[1][ends] == w[1]).all()
    assert (keys.decrypt(got) == numpy.where(bits[0], bits[1], bits[2])).all()
