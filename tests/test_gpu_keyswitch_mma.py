"""The tensor-core key switch (keyswitch_mma_kernel, nb_ks_prepare) against the gather kernel and the CPU oracle.

Two engines share the device: one with NUFHE_B200_KS_MMA_MIN=1 (every batch of a prepared key takes the GEMM), one with
a threshold no batch reaches (every batch takes keyswitch_kernel).  Both must give the same (a, b, variance) bits."""
import functools
import os

import numpy
import pytest

import gen_inputs as G
from oracle import oracle as O

pytestmark = pytest.mark.gpu

BATCHES = (1, 31, 32, 33, 127, 128, 129, 256, 1000, 4096, 4097, 16384)


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
    return _engine(1), _engine(1 << 62)


@functools.lru_cache(maxsize=None)
def _keys(kind):
    """host (ks_a, ks_b, ks_cv) of the given kind; d = 0 rows zero except for 'pad'"""
    rng = G.rs(31)
    if kind == 'generated':
        return O.OracleKeys(G.GATE_SEED).ks
    ks_a = G.torus32(rng, (1024, 8, 4, 500))
    ks_b = G.torus32(rng, (1024, 8, 4))
    ks_cv = rng.uniform(0.0, 1e-6, size=(1024, 8, 4)).astype(numpy.float32)
    if kind == 'bytes_ff':
        ks_a[:] = -1
        ks_b[:] = -1
    elif kind == 'min_word':
        ks_a[:] = -2**31
        ks_b[:] = -2**31
    if kind != 'pad':
        ks_a[:, :, 0] = 0
        ks_b[:, :, 0] = 0
    return ks_a, ks_b, ks_cv


def _run_both(engs, host_ks, srcs, c=0):
    gemm, gather = engs
    out = []
    for eng, prepare in ((gemm, True), (gather, False)):
        ks = tuple(eng.to_device(x) for x in host_ks)
        planes = eng.ks_prepare(ks[0], ks[1]) if prepare else None
        dev = [(eng.to_device(a), eng.to_device(b)) for a, b in srcs]
        ra, rb, rcv = eng.keyswitch(ks, dev[0], dev[1] if len(dev) > 1 else None, c=c, want_cv=True)
        out.append((eng.to_host(ra), eng.to_host(rb), eng.to_host(rcv)))
        del planes
    return out


def _same(x, y):
    for u, v in zip(x, y):
        assert u.shape == v.shape and (u.view(numpy.uint32) == v.view(numpy.uint32)).all()


@pytest.mark.parametrize('kind', ['generated', 'bytes_ff', 'min_word', 'pad'])
def test_paths_agree(engs, kind):
    host_ks = _keys(kind)
    gemm = engs[0]
    ks = tuple(gemm.to_device(x) for x in host_ks)
    planes = gemm.ks_prepare(ks[0], ks[1])
    assert (planes is None) == (kind == 'pad')        # non-zero d = 0 rows stay on the gather kernel
    del planes
    rng = G.rs(32)
    for B in BATCHES:
        src = (G.torus32(rng, (B, 1024)), G.torus32(rng, (B,)))
        if kind in ('bytes_ff', 'min_word'):
            src[0][:] = -1 - 2**15                   # all digits 3: 8192 one-hot columns, the largest plane sums
        x, y = _run_both(engs, host_ks, [src])
        _same(x, y)
        idx = numpy.unique(numpy.linspace(0, B - 1, min(B, 6)).astype(int))
        wa, wb, _ = O.lwe_keyswitch(*host_ks, src[0][idx], src[1][idx])
        assert (x[0][idx] == wa).all() and (x[1][idx] == wb).all(), B


def test_mux_fold(engs):
    """src1 + src2 + (0, c), as gate_mux calls it"""
    host_ks = _keys('generated')
    rng = G.rs(33)
    for B in (1, 129, 4097):
        s1 = (G.torus32(rng, (B, 1024)), G.torus32(rng, (B,)))
        s2 = (G.torus32(rng, (B, 1024)), G.torus32(rng, (B,)))
        x, y = _run_both(engs, host_ks, [s1, s2], c=2**29)
        _same(x, y)
        with numpy.errstate(over='ignore'):
            sa = (s1[0][:5] + s2[0][:5]).astype(numpy.int32)
            sb = (s1[1][:5] + s2[1][:5] + numpy.int32(2**29)).astype(numpy.int32)
        wa, wb, _ = O.lwe_keyswitch(*host_ks, sa, sb)
        assert (x[0][:5] == wa).all() and (x[1][:5] == wb).all()


def test_golden_on_the_gemm(engs, golden):
    g = golden('keyswitch')
    ks_a, ks_b, ks_cv, src_a, src_b = G.keyswitch_inputs()
    eng = engs[0]
    ks = (eng.to_device(ks_a), eng.to_device(ks_b), eng.to_device(ks_cv))
    planes = eng.ks_prepare(ks[0], ks[1])
    assert planes is not None
    ra, rb, rcv = eng.keyswitch(ks, (eng.to_device(src_a), eng.to_device(src_b)), want_cv=True)
    assert (eng.to_host(ra) == g['res_a']).all() and (eng.to_host(rb) == g['res_b']).all()
    assert numpy.allclose(eng.to_host(rcv), g['res_cv'], rtol=1e-4, atol=1e-4)


def test_registration_follows_the_planes(engs):
    """freeing the planes drops the registration: the same key then runs the gather kernel, with the same bits"""
    eng = engs[0]
    host_ks = _keys('generated')
    ks = tuple(eng.to_device(x) for x in host_ks)
    rng = G.rs(34)
    src = (eng.to_device(G.torus32(rng, (300, 1024))), eng.to_device(G.torus32(rng, (300,))))
    planes = eng.ks_prepare(ks[0], ks[1])
    first = [eng.to_host(x) for x in eng.keyswitch(ks, src, want_cv=True)]
    planes.zero_()                                   # the GEMM reads the planes: zeroed planes give other bits
    spoiled = eng.to_host(eng.keyswitch(ks, src)[0])
    assert not (spoiled == first[0]).all()
    del planes
    again = [eng.to_host(x) for x in eng.keyswitch(ks, src, want_cv=True)]
    _same(first, again)
