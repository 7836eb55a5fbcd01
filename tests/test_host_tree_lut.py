"""Tree-based programmable bootstrapping on the CPU: the key switch and assembly of csrc/tree_layout.cuh (through the
host emulator's scalar models of plane_gemm_kernel and tree_assemble_kernel) against the NumPy restatement
(tree_ref.py), the tree key (draw order, row phases, pickles), the noise rule, and vm.lut_tree end to end on an
oracle-backed engine double."""
import ctypes
import io
import os

import numpy
import pytest

import nufhe_b200
from nufhe_b200 import lut, tree_lut
from nufhe_b200.compressed import draw_seed
from nufhe_b200.packing import PACK_GADGET, PACK_LEVELS
from nufhe_b200.random_numbers import DeterministicRNG
from chacha_ref import seeded_uniform
from fake_engine import _np, _t
from oracle import oracle as O
from test_host_lut import LutFakeEngine
import pack_ref
import tree_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 1024
SIGMA = 9e-9 * (2 / numpy.pi)**0.5


@pytest.fixture(scope='module')
def emul():
    path = os.path.join(ROOT, 'nufhe_b200', 'csrc', 'libnb_host_emul.so')
    if not os.path.exists(path):
        import __graft_entry__ as g
        g.build()
    lib = ctypes.CDLL(path)
    lib.emul_tree_keyswitch.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p,
                                                                ctypes.c_size_t]
    lib.emul_tree_keyswitch.restype = None
    lib.emul_tree_assemble.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                       ctypes.c_size_t]
    lib.emul_tree_assemble.restype = None
    return lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _rand(rng, shape):
    return rng.randint(-2**31, 2**31, size=shape, dtype=numpy.int64).astype(numpy.int32)


def _emul_keyswitch(emul, a, masks, body):
    R, n = a.shape
    k = masks.shape[2]
    out = numpy.empty((R, k + 1, N), numpy.int32)
    emul.emul_tree_keyswitch(_p(a), _p(masks), _p(body), n, k, _p(out), R)
    return out


def test_exactness_bound():
    """Every plane sum of the key switch is at most kpad * 128 * 255 < 2^31 (kpad = n t rounded up to 32)."""
    for k in (1, 2):
        params = nufhe_b200.NuFHEParameters(tlwe_mask_size=k)
        n = params.in_out_params.size
        kpad = -(-n * PACK_LEVELS // 32) * 32
        assert kpad == 1024 and kpad * 128 * 255 < 2**31
    assert PACK_GADGET == (2**24, 2**16)


@pytest.mark.parametrize('rows,k,n', [(1, 1, 500), (15, 2, 500), (16, 1, 500), (17, 1, 37), (129, 2, 20)])
def test_keyswitch_emulator_matches_restatement(emul, rows, k, n):
    rng = numpy.random.RandomState(rows * 10 + k)
    a = _rand(rng, (rows, n))
    a[0, :4] = [0, -1, 2**31 - 1, -2**31]
    masks, body = _rand(rng, (n, 2, k, N)), _rand(rng, (n, 2, N))
    assert (_emul_keyswitch(emul, a, masks, body) == tree_ref.keyswitch(a, masks, body)).all()


def test_keyswitch_at_the_exactness_bound(emul):
    """All digits -128 (mask words 0x7f7f8000) and all key words -2^31: every plane sum is at its extreme."""
    n = 500
    a = numpy.full((16, n), 0x7f7f8000, numpy.int64).astype(numpy.int32)
    assert (pack_ref.digits(a) == -128).all()
    masks = numpy.full((n, 2, 1, N), -2**31, numpy.int32)
    body = numpy.full((n, 2, N), -2**31, numpy.int32)
    want = tree_ref.keyswitch(a, masks, body)
    assert (want == 0).all()                         # 2000 * 128 * 2^31 = 0 mod 2^32
    assert (_emul_keyswitch(emul, a, masks, body) == want).all()
    masks[:, :, :, 1::2] = 2**31 - 1
    body[:, :, ::3] = 1
    assert (_emul_keyswitch(emul, a, masks, body) == tree_ref.keyswitch(a, masks, body)).all()


@pytest.mark.parametrize('bits', [1, 2])
@pytest.mark.parametrize('k', [1, 2])
def test_assemble_emulator_matches_restatement(emul, bits, k):
    rng = numpy.random.RandomState(bits + 3 * k)
    T, M = 3, 1 << bits
    v, b = _rand(rng, (T, M, k + 1, N)), _rand(rng, (T, M))
    got = numpy.empty((T, k + 1, N), numpy.int32)
    emul.emul_tree_assemble(_p(v), _p(b), bits, k, _p(got), T)
    assert (got == tree_ref.assemble(v, b, bits)).all()
    # a trivial GLWE (zero masks, body = the encodings at X^0) assembles to make_test_vector
    table = rng.randint(0, M, size=M)
    v = numpy.zeros((1, M, k + 1, N), numpy.int32)
    b = lut.encode_int(table, bits)[None]
    emul.emul_tree_assemble(_p(v), _p(b), bits, k, _p(got[:1]), 1)
    assert (got[0, :k] == 0).all() and (got[0, k] == lut.make_test_vector(table, bits)).all()


# ---------------------------------------------------------------- keys

class TreeFakeEngine(LutFakeEngine):
    """LutFakeEngine plus Engine.seeded_uniform from the NumPy keystream, the two tree steps from tree_ref, and the
    encrypted-test-vector bootstrap composed from the oracle's steps."""

    def seeded_uniform(self, seed, nonce, shape, first=0):
        return _t(seeded_uniform(seed, nonce, shape, first))

    def tree_prepare(self, masks, body):
        return (masks, body)

    def tree_keyswitch(self, a, planes, mask_size):
        self._count('tree_keyswitch')
        return _t(tree_ref.keyswitch(_np(a), _np(planes[0]), _np(planes[1])))

    def tree_assemble(self, v, b, bits):
        self._count('tree_assemble')
        return _t(tree_ref.assemble(_np(v), _np(b), bits))

    def bootstrap_glwe_lut_extract(self, x, tv, bk_int):
        self._count('bootstrap_glwe_lut_extract')
        a, b = _np(x[0]), _np(x[1])
        B = b.size
        barb = O.t32_to_phase(b.reshape(B), 2 * N).astype(numpy.int32)
        bara = O.t32_to_phase(a.reshape(B, -1), 2 * N).astype(numpy.int32)
        acc = O.shift_torus_polynomial(_np(tv).reshape(B, 2, N), barb, invert_powers=True)
        acc = O.blind_rotate(acc, _np(bk_int, True), bara)
        ea, eb = O.tlwe_extract_lwe_samples(acc)
        return _t(ea), _t(eb)


def _context(seed):
    return nufhe_b200.Context(rng=DeterministicRNG(seed), thread=TreeFakeEngine())


@pytest.fixture(scope='module')
def keys():
    ctx = _context(71)
    sk = ctx.make_secret_key()
    ck, tk = ctx.make_cloud_key(sk, tree_key=True)
    return ctx, sk, ck, tk


def _glwe_key(seed, k=1):
    replay = DeterministicRNG(seed)
    replay.uniform_bool((500,))
    return replay.uniform_bool((k, N))                   # the TGSW key's TLWE key, drawn first by make_cloud_key


def _key_polys(tk):
    k = tk.params.tgsw_params.tlwe_params.mask_size
    return pack_ref.key_polys(seeded_uniform(tk.seed, tree_lut.NONCE_TREE_KEY, (500, PACK_LEVELS, k, N)), _np(tk.body))


def test_draw_order_and_cloud_key_unchanged(keys):
    ctx, sk, ck, tk = keys
    ctx2 = _context(71)
    sk2 = ctx2.make_secret_key()
    ck2 = ctx2.make_cloud_key(sk2)
    assert sk2 == sk and ck2 == ck and ck2.dumps() == ck.dumps()
    assert (draw_seed(ctx2.rng) == tk.seed).all()        # the tree key's seed is the next draw
    assert isinstance(tk, nufhe_b200.NuFHETreeKey) and not isinstance(tk, nufhe_b200.NuFHEPackingKey)
    assert tuple(tk.body.shape) == (500, PACK_LEVELS, N) and tk.variance == float(numpy.float32(SIGMA**2))
    # compressed: the same
    c1, c2 = _context(72), _context(72)
    s1, s2 = c1.make_secret_key(), c2.make_secret_key()
    cck, ctk = c1.make_cloud_key(s1, compressed=True, tree_key=True)
    cck2 = c2.make_cloud_key(s2, compressed=True)
    assert cck == cck2 and cck.dumps() == cck2.dumps()
    assert (draw_seed(c2.rng) == ctk.seed).all()


def test_tree_key_row_phases(keys):
    ctx, sk, ck, tk = keys
    S = _glwe_key(71)
    K = _key_polys(tk)                                   # (n t, 2, N)
    phase = tree_ref.glwe_phase(K, S).astype(numpy.int64)
    s = _np(sk.lwe_key.key).astype(numpy.int64)
    msg = numpy.zeros((500 * PACK_LEVELS, N), numpy.int64)
    msg[:, 0] = (s[:, None] * numpy.array(PACK_GADGET)[None, :]).reshape(-1)
    err = pack_ref.i32(phase - msg).astype(numpy.int64)
    assert numpy.abs(err).max() < 8 * SIGMA * 2**32
    assert err.std() > 0.5 * SIGMA * 2**32


def test_pickles_and_types(keys):
    ctx, sk, ck, tk = keys
    s = tk.dumps()
    assert ctx.load_tree_key(s) == tk and ctx.load_tree_key(io.BytesIO(s)) == tk
    psk, pk = ctx.make_packing_keys(sk)
    for wrong in (pk.dumps(), sk.dumps(), b'junk'):
        with pytest.raises(ValueError):
            ctx.load_tree_key(wrong)
    with pytest.raises(ValueError):
        ctx.load_packing_key(s)
    vm = ctx.make_virtual_machine(ck)
    t = vm.make_tree_lut(numpy.zeros((4, 4), int), bits=2, digits=2)
    d = ctx.encrypt_int(sk, [0], 2)
    for wrong in (pk, ck, None):
        with pytest.raises(TypeError):
            vm.lut_tree(wrong, t, [d, d])


def test_assembled_test_vector_decrypts(keys):
    ctx, sk, ck, tk = keys
    S = _glwe_key(71)
    rng = numpy.random.RandomState(3)
    params = sk.params
    for bits in (1, 2):
        M = 1 << bits
        table = rng.randint(0, M, size=(2, M))
        ct = ctx.encrypt_int(sk, table, bits)                  # (2, M)
        v = tree_ref.keyswitch(_np(ct.a).reshape(-1, 500), *(_np(x) for x in (tk.masks(ctx.thread), tk.body)))
        tv = tree_ref.assemble(v.reshape(2, M, 2, N), _np(ct.b).reshape(2, M), bits)
        err = pack_ref.i32(tree_ref.glwe_phase(tv, S).astype(numpy.int64)
                           - lut.make_test_vector(table, bits).astype(numpy.int64)).astype(numpy.int64)
        sigma = (params.in_out_params.min_noise**2 + tree_lut.test_vector_variance(params, bits))**0.5
        assert numpy.abs(err).max() < 8 * sigma * 2**32, bits


def test_noise_rule():
    params = nufhe_b200.NuFHEParameters()
    for bits in (1, 2):
        derived = max(d for d in range(1, tree_lut.MAX_DIGITS + 1)
                      if 2.0**-(bits + 2) / tree_lut.tree_sigma(params, bits, d) >= lut.MARGIN_SIGMAS)
        assert tree_lut.max_digits(params, bits) == derived
    assert tree_lut.max_digits(params, 2) == 4
    assert abs(tree_lut.test_vector_variance(params, 2) - 7.7e-8) < 0.2e-8
    # the estimate-only margins of DESIGN.md section 13 at P = 2
    blind_ks = lut._sigma_estimate(params.in_out_params, params.tgsw_params, params.ks_decomp_length,
                                   params.ks_log2_base, 0, None)**2 - tree_lut._modswitch_variance(params)
    assert abs(blind_ks - 1.28e-5) < 0.01e-5
    for d, want in ((2, 11.3), (3, 9.5), (4, 8.3), (6, 6.9)):
        var = d * blind_ks + (d - 1) * tree_lut.test_vector_variance(params, 2) + tree_lut._modswitch_variance(params)
        assert abs(0.0625 / var**0.5 - want) < 0.15, d
    for bad in (dict(bits=3, digits=2), dict(bits=2, digits=1), dict(bits=2, digits=5)):
        with pytest.raises(ValueError):
            tree_lut._check_config(params, **bad)


# ---------------------------------------------------------------- lut_tree on the double

def _all_inputs(bits, D):
    M = 1 << bits
    grid = numpy.stack(numpy.meshgrid(*[numpy.arange(M)] * D, indexing='ij'), -1).reshape(-1, D)
    return [grid[:, i] for i in range(D)]                  # d_{D-1}, ..., d_0


@pytest.mark.parametrize('bits,D', [(2, 2), (1, 3)])
def test_lut_tree_all_inputs_fused_and_steps(keys, bits, D):
    ctx, sk, ck, tk = keys
    thr = ctx.thread
    M = 1 << bits
    rng = numpy.random.RandomState(bits * 10 + D)
    tables = rng.randint(0, M, size=(2,) + (M,) * D)
    values = _all_inputs(bits, D)
    digits = [ctx.encrypt_int(sk, v, bits) for v in values]
    vm_fused = ctx.make_virtual_machine(ck)
    vm_steps = ctx.make_virtual_machine(ck, perf_params=nufhe_b200.PerformanceParameters(
        ck.params, single_kernel_bootstrap=False))
    want = tables[(slice(None),) + tuple(values)]           # (F, combos)
    results = []
    for vm, counter in ((vm_fused, 'bootstrap_glwe_lut_extract'), (vm_steps, 'shift_torus_polynomial')):
        before = thr.calls.get(counter, 0)
        out = vm.lut_tree(tk, vm.make_tree_lut(tables, bits, D), digits)
        assert thr.calls.get(counter, 0) > before
        for f in range(2):
            assert (ctx.decrypt_int(sk, out[f], bits) == want[f]).all(), (vm is vm_steps, f)
        results.append(out)
    for r_f, r_s in zip(*results):
        assert (_np(r_f.a) == _np(r_s.a)).all() and (_np(r_f.b) == _np(r_s.b)).all()
    # one function, gate-compatible bits
    t = vm_fused.make_tree_lut(tables[0] % 2, bits, D, out='bool')
    r = vm_fused.lut_tree(tk, t, digits)
    assert isinstance(r, nufhe_b200.LweSampleArray)
    assert (ctx.decrypt(sk, r) == (want[0] % 2 == 1)).all()


def test_lut_tree_errors(keys):
    ctx, sk, ck, tk = keys
    vm = ctx.make_virtual_machine(ck)
    t = vm.make_tree_lut(numpy.zeros((4, 4), int), bits=2, digits=2)
    d2, d3 = ctx.encrypt_int(sk, [0, 1], 2), ctx.encrypt_int(sk, [0, 1, 2], 2)
    with pytest.raises(ValueError):
        vm.lut_tree(tk, t, [d2])
    with pytest.raises(ValueError):
        vm.lut_tree(tk, t, [d2, d3])
    for bad in (dict(bits=3, digits=2), dict(bits=2, digits=1), dict(bits=2, digits=5)):
        with pytest.raises(ValueError):
            vm.make_tree_lut(numpy.zeros((1 << bad['bits'],) * bad['digits'], int), **bad)
    with pytest.raises(ValueError):
        vm.make_tree_lut(numpy.zeros((4, 4, 3), int), bits=2, digits=2)
    other = tree_lut.NuFHETreeKey(nufhe_b200.NuFHEParameters(tlwe_mask_size=2), tk.seed, tk.body, tk.variance)
    with pytest.raises(ValueError):
        vm.lut_tree(other, t, [d2, d2])
