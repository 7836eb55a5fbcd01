"""Encrypted-index lookups on the CPU (DESIGN.md section 15): the oracle-composed reference (tests/index_ref.py) against
the noiseless-selector identity, the per-slot-key FP64 step of the kernels (host emulator) against the reference bit
for bit, and the Python layer on the oracle-backed engine double: draws, pickles, compressed selectors, argument errors
and the noise estimates."""
import copy
import ctypes
import os

import numpy
import pytest
import torch

import index_ref as R
from fake_engine import FakeEngine
from oracle import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 1024


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


# ---- the reference ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('m, W', [(1, 1), (4, 1), (9, 1), (10, 1), (11, 1), (13, 1), (8, 4), (3, 100), (11, 3), (10, 2)])
def test_noiseless_selectors_look_up_exactly(m, W):
    """trivial selectors b H and a table of multiples of 2^12: the reference returns exactly (0, table[w][idx]) for
    every idx (1 024 of them, the first and last included, when the table has more than 2^11 entries), W > 1 on both
    sides of m = 10"""
    rng = numpy.random.RandomState(m * 100 + W)
    enc = (rng.randint(0, 2**20, size=(W, 1 << m)).astype(numpy.int64) << 12).astype(numpy.uint32).view(numpy.int32)
    if W << m <= 2048:
        idx = numpy.arange(1 << m)
    else:
        idx = numpy.concatenate([[0, (1 << m) - 1], rng.randint(0, 1 << m, size=1022)])
    bits = (idx[:, None] >> numpy.arange(m)) & 1
    # two distinct rows per bit: row 2 j + b is selector j with value b
    sel = R.noiseless_selectors(numpy.stack([numpy.zeros(m, int), numpy.ones(m, int)], 1))     # (m, 2, ...)
    rows = 2 * numpy.arange(m)[None, :] + bits
    a, b = R.lookup(R.table_polys(enc, m), R.transform(sel), rows, m, W)
    assert (a == 0).all()
    assert numpy.array_equal(b, enc[:, idx])


# ---- the kernels' step on the host -----------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def emul():
    return ctypes.CDLL(os.path.join(ROOT, 'nufhe_b200', 'csrc', 'libnb_host_emul.so'))


def _slots(emul, acc, rows_ref, rot):
    out = numpy.ascontiguousarray(acc.copy())
    rp = None if rot is None else _p(numpy.ascontiguousarray(rot, numpy.int32))
    assert emul.emul_fft_step_slots(_p(out), _p(numpy.ascontiguousarray(rows_ref)), rp) == 0
    return out


@pytest.mark.parametrize('case', ['random', 'worst'])
def test_emulated_step_with_a_row_per_slot_matches_reference(emul, case):
    """the FP64 step of the index kernels (fwd1, fwd2, pass 3 with each slot's own key row, inv2, inv1; host
    emulator) with two different rows in the two slots: the plain product (CMux level) and the rotation step, against
    the oracle's external product bit for bit, for random rows and for rows at the extremes of the 32-bit range with
    digits at -512 / 511"""
    rng = numpy.random.RandomState(5 if case == 'random' else 6)
    if case == 'random':
        raw = rng.randint(-2**31, 2**31, size=(2, 2, 2, 2, N), dtype=numpy.int64).astype(numpy.int32)
        acc = rng.randint(-2**31, 2**31, size=(2, 2, N), dtype=numpy.int64).astype(numpy.int32)
    else:
        raw = numpy.empty((2, 2, 2, 2, N), numpy.int64)
        pats = [numpy.full(N, -2**31), numpy.full(N, 2**31 - 1), numpy.where(numpy.arange(N) % 2, -2**31, 2**31 - 1),
                numpy.full(N, -2**31 + 2**15), numpy.full(N, 2**15 - 1)]
        for i, ix in enumerate(numpy.ndindex(2, 2, 2, 2)):
            raw[ix] = pats[i % len(pats)]
        raw = raw.astype(numpy.int32)
        lo = numpy.int64(-(2**31 + 2**21)) & 0xffffffff
        hi = (numpy.int64(0xfffff000) - (2**31 + 2**21)) & 0xffffffff
        acc = numpy.empty((2, 2, N), numpy.int64)
        acc[0, 0], acc[0, 1] = lo, hi
        acc[1] = numpy.where(numpy.arange(N) % 2, lo, hi)
        acc = acc.astype(numpy.uint32).view(numpy.int32)
    ref = R.transform(raw)
    rows = numpy.array([0, 1])
    got = _slots(emul, acc, ref, None)
    want = R.apply(acc[:, None], ref, rows)[:, 0]
    assert numpy.array_equal(got, want)
    for j in (0, 5, 9):
        rot = numpy.full(2, 2 * N - (1 << j))
        got = _slots(emul, acc, ref, rot)
        tmp = O.shift_torus_polynomial(acc, rot.astype(numpy.int32), minus_one=True)
        want = R.add(acc, R.apply(tmp[:, None], ref, rows)[:, 0])
        assert numpy.array_equal(got, want)


# ---- the Python layer on the engine double ---------------------------------------------------------------------------

@pytest.fixture(scope='module')
def nufhe():
    import nufhe_b200
    return nufhe_b200


class _SeededFakeEngine(FakeEngine):
    """the engine double with Engine.seeded_uniform from the NumPy keystream (compressed keys and selectors)"""

    def seeded_uniform(self, seed, nonce, shape, first=0):
        from chacha_ref import seeded_uniform
        return torch.from_numpy(numpy.ascontiguousarray(seeded_uniform(seed, nonce, shape, first)))


def _ctx(nufhe, seed):
    return nufhe.Context(rng=nufhe.DeterministicRNG(seed), thread=_SeededFakeEngine())


@pytest.fixture(scope='module')
def keys(nufhe):
    ctx = _ctx(nufhe, 91)
    sk = ctx.make_secret_key()
    ck, ik = ctx.make_cloud_key(sk, index_key=True)
    return ctx, sk, ck, ik


@pytest.mark.parametrize('compressed, multi_bit', [(False, 1), (True, 1), (True, 2)])
def test_index_key_draws_nothing(nufhe, compressed, multi_bit):
    """index_key=True leaves the cloud key and a tree key made in the same call byte-identical, and returns S"""
    ctx1, ctx2 = _ctx(nufhe, 92), _ctx(nufhe, 92)
    sk1, sk2 = ctx1.make_secret_key(), ctx2.make_secret_key()
    ck1, tk1 = ctx1.make_cloud_key(sk1, compressed=compressed, tree_key=True, multi_bit=multi_bit)
    ck2, tk2, ik = ctx2.make_cloud_key(sk2, compressed=compressed, tree_key=True, multi_bit=multi_bit, index_key=True)
    assert ck1.dumps() == ck2.dumps() and tk1.dumps() == tk2.dumps()
    assert ctx1.rng.rng.randint(2**31) == ctx2.rng.rng.randint(2**31)
    assert isinstance(ik, nufhe.NuFHEIndexSecretKey) and tuple(ik.key.shape) == (1, N)


def _phases(sel, S):
    """the phases body - S mask of selector rows (..., 2, 2, 2, N), as (..., 2, 2, N) int64 centred"""
    c = numpy.ascontiguousarray(sel).reshape(-1, 2, 2, 2, N)
    mask = numpy.ascontiguousarray(c[:, :, :, 0]).reshape(-1, N)
    prod = O.poly_mul_i32(S, mask).reshape(c.shape[0], 2, 2, N)
    ph = (c[:, :, :, 1].astype(numpy.int64) - prod.astype(numpy.int64)) & 0xffffffff
    return numpy.where(ph >= 2**31, ph - 2**32, ph)


def _check_selectors(sel, S, values, m):
    c = numpy.ascontiguousarray(sel).reshape(-1, 2, 2, 2, N)
    bits = ((numpy.asarray(values).reshape(-1, 1) >> numpy.arange(m)) & 1).reshape(-1)
    ph = _phases(c, S)
    # row (mi = 1, j): phase b 2^(22 - 10 j) X^0 + noise
    want = numpy.zeros((c.shape[0], 2, N), numpy.int64)
    want[:, 0, 0] = bits << 22
    want[:, 1, 0] = bits << 12
    assert numpy.abs(ph[:, 1] - want).max() < 2**10
    # row (mi = 0, j): the mask carries b h_j, so the phase is -b h_j S + noise
    Sl = S.astype(numpy.int64)
    want0 = -(bits[:, None, None] * numpy.array([2**22, 2**12])[None, :, None]) * Sl[None, None, :]
    d = (ph[:, 0] - want0 + 2**31) % 2**32 - 2**31
    assert numpy.abs(d).max() < 2**10


def test_selectors_encrypt_the_index_bits(nufhe, keys):
    ctx, sk, ck, ik = keys
    values = numpy.array([[0, 5], [31, 17]])
    e = ctx.encrypt_index(ik, values, 5)
    assert isinstance(e, nufhe.EncryptedIndexArray) and e.shape == (2, 2) and e.bits == 5
    assert tuple(e.samples.shape) == (2, 2, 5, 2, 2, 2, N)
    _check_selectors(e.samples.numpy(), ik.key.numpy()[0], values, 5)


def test_compressed_selectors_expand_to_the_same_samples(nufhe, keys):
    """compressed: a seed and the bodies; decompress() regenerates the masks from ChaCha20 (seed, nonce 6), and the
    samples decrypt to the same bits; the draws are the seed, then the body noises"""
    from chacha_ref import seeded_uniform
    from nufhe_b200.index_lookup import NONCE_INDEX
    ctx, sk, ck, ik = keys
    values = numpy.array([3, 0, 7])
    c = ctx.encrypt_index(ik, values, 3, compressed=True)
    assert isinstance(c, nufhe.CompressedEncryptedIndexArray) and tuple(c.body.shape) == (3, 3, 2, 2, N)
    d = c.decompress(ctx.thread)
    s = d.samples.numpy()
    assert numpy.array_equal(s[..., 0, :].reshape(-1), seeded_uniform(c.seed, NONCE_INDEX, (9, 2, 2, 1, N)).reshape(-1))
    assert numpy.array_equal(s[..., 1, :], c.body.numpy())
    _check_selectors(s, ik.key.numpy()[0], values, 3)
    assert c.decompress(ctx.thread) == d


def test_pickles_round_trip(nufhe, keys):
    ctx, sk, ck, ik = keys
    e = ctx.encrypt_index(ik, [1, 2], 2)
    c = ctx.encrypt_index(ik, [1, 2], 2, compressed=True)
    assert ctx.load_index_secret_key(ik.dumps()) == ik
    assert ctx.load_encrypted_index(e.dumps()) == e
    assert ctx.load_encrypted_index(c.dumps()) == c
    assert b'nufhe_b200.EncryptedIndexArray/1' in e.dumps()
    for wrong in (sk.dumps(), ik.dumps(), b'not a pickle'):
        with pytest.raises(ValueError):
            ctx.load_encrypted_index(wrong)
    with pytest.raises(ValueError):
        ctx.load_index_secret_key(e.dumps())
    with pytest.raises(ValueError):
        nufhe.EncryptedIndexArray.loads(c.dumps(), ctx.thread)


def test_argument_errors(nufhe, keys):
    from nufhe_b200 import index_lookup as IL
    ctx, sk, ck, ik = keys
    for bits in (0, 21, 2.5):
        with pytest.raises(ValueError):
            ctx.encrypt_index(ik, [0], bits)
    for values, bits in (([-1], 3), ([8], 3), ([1 << 20], 20), ([0.5], 2)):
        with pytest.raises(ValueError):
            ctx.encrypt_index(ik, values, bits)
    with pytest.raises(TypeError):
        ctx.encrypt_index(sk, [0], 2)
    # tlwe_mask_size = 2
    ctx2 = _ctx(nufhe, 93)
    sk2 = ctx2.make_secret_key(tlwe_mask_size=2)
    with pytest.raises(ValueError):
        ctx2.make_cloud_key(sk2, index_key=True)
    # tables
    thr = ctx.thread
    for table, kw in ((numpy.zeros(3), {'out': 'bool'}), (numpy.zeros((5, 256)), {'out': 'bool'}),
                      (numpy.zeros(1 << 21), {'out': 'bool'}), (numpy.zeros(8), {'out': 'float'}),
                      (numpy.zeros(8), {'out': 'int'}), (numpy.full(8, 4), {'out': 'int', 'bits': 2})):
        with pytest.raises(ValueError):
            IL.IndexTable(thr, sk.params, table, **kw)
    t = IL.IndexTable(thr, sk.params, numpy.arange(8) % 4, out='int', bits=2)
    assert tuple(t.polys.shape) == (1, 2, N) and t.single and t.columns == 1
    e = ctx.encrypt_index(ik, [1, 2], 3)
    c = ctx.encrypt_index(ik, [1, 2], 3, compressed=True)
    ks = ck.keyswitch_key
    with pytest.raises(TypeError):
        IL.lookup(thr, ks, c, t)
    with pytest.raises(TypeError):
        IL.lookup(thr, ks, sk, t)
    with pytest.raises(TypeError):
        IL.lookup(thr, ks, e, numpy.arange(8))
    with pytest.raises(ValueError):
        IL.lookup(thr, ks, ctx.encrypt_index(ik, [1], 4), t)
    t_other = IL.IndexTable(thr, copy.deepcopy(sk.params), numpy.arange(8) % 4, out='int', bits=2)
    t_other.params._tlwe_mask_size = 2                 # a table made for other parameters
    assert t_other.params != e.params
    with pytest.raises(ValueError):
        IL.lookup(thr, ks, e, t_other)


def test_table_layouts(nufhe, keys):
    """m < 10: all columns in one polynomial at i + w 2^m; m >= 10: 2^(m-10) polynomials per column"""
    from nufhe_b200 import index_lookup as IL
    from nufhe_b200.gates import MU
    ctx, sk, ck, ik = keys
    tab = numpy.arange(4 * 256).reshape(4, 256) % 4
    t = IL.IndexTable(ctx.thread, sk.params, tab, out='int', bits=2)
    assert numpy.array_equal(t.polys.numpy(), R.table_polys(tab.astype(numpy.int32) << 29, 8))
    tab = numpy.arange(2 * 2048).reshape(2, 2048) % 2
    t = IL.IndexTable(ctx.thread, sk.params, tab, out='bool')
    assert tuple(t.polys.shape) == (4, 2, N) and not t.single
    enc = numpy.where(tab != 0, int(MU), -int(MU)).astype(numpy.int32)
    assert numpy.array_equal(t.polys.numpy(), R.table_polys(enc, 11))
    assert IL.queries_per_pass(20, 1) * (20 * 2**17 + 2**10 * 8192) <= IL.PASS_BYTES


def test_noise_estimates(nufhe):
    """m x 1.84e-8 (selector noise; the rounded decomposition adds 3.9e-11 per CMux) plus the key switch's 3.6e-6:
    4.0e-6 (sigma 2.0e-3) at m = 20, below a gate output's 1.28e-5, and every table within the caps keeps more than
    7 sigma for bool outputs and for int outputs of up to 3 bits"""
    from nufhe_b200 import index_lookup as IL
    params = nufhe.NuFHEParameters()
    assert IL.cmux_variance(params) == pytest.approx(1.84e-8, rel=0.01)
    assert IL.decomposition_variance(params) == pytest.approx(3.9e-11, rel=0.01)
    assert IL.keyswitch_variance(params) == pytest.approx(3.6e-6, rel=0.02)
    assert IL.extracted_variance(params, 16) == pytest.approx(16 * 1.85e-8, rel=0.01)
    assert IL.output_variance(params, 20) == pytest.approx(4.01e-6, rel=0.01)
    assert IL.output_sigma(params, 20) == pytest.approx(2.0e-3, rel=0.01)
    assert IL.output_variance(params, 20) < 1.28e-5
    for m in range(1, IL.MAX_BITS + 1):
        s = IL.output_sigma(params, m)
        assert 1 / 8 / s > 7
        for P in (1, 2, 3):
            assert 2.0**-(P + 2) / s > 7
