"""Programmable bootstrapping on the CPU: the integer encoding, the test-vector layout (nufhe_b200/lut.py), the kernel's
head and tail index functions run by the host emulator (csrc/lut_index.cuh via host_emul.cpp) against the oracle's
steps, the noise table, and the Python layer end to end on an oracle-backed engine double."""
import ctypes
import os

import numpy
import pytest
import torch

import gen_inputs as G
from fake_engine import FakeEngine, _np, _t
from oracle import oracle as O
from nufhe_b200 import lut

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 1024


@pytest.fixture(scope='module')
def emul():
    path = os.path.join(ROOT, 'nufhe_b200', 'csrc', 'libnb_host_emul.so')
    if not os.path.exists(path):
        import __graft_entry__ as g
        g.build()
    lib = ctypes.CDLL(path)
    lib.emul_modswitch_lut.argtypes = [ctypes.c_int32, ctypes.c_int]
    return lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def test_encode_decode_round_trip():
    for bits in (1, 2, 3):
        m = numpy.arange(2**bits)
        enc = lut.encode_int(m, bits)
        assert (enc.astype(numpy.int64) == m * 2**(31 - bits)).all()
        assert (lut.decode_int(enc, bits) == m).all()
        # anything inside the box decodes to the box's message, including m = 0 from below
        half = 2**(30 - bits)
        for off in (-half + 1, -1, 1, half - 1):
            noisy = ((enc.astype(numpy.int64) + off) & 0xffffffff).astype(numpy.uint32).view(numpy.int32)
            assert (lut.decode_int(noisy, bits) == m).all()
    with pytest.raises(ValueError):
        lut.encode_int([4], 2)
    with pytest.raises(ValueError):
        lut.encode_int([0], 4)


def _rotate_coef(tv, b, j):
    """coefficient j of X^(-b) * tv (negacyclic)"""
    i = (b + j) % (2 * N)
    return tv[i] if i < N else -int(tv[i - N])


@pytest.mark.parametrize('bits', [1, 2, 3])
def test_test_vector_boxes_exhaustive(bits):
    rng = numpy.random.RandomState(bits)
    M, box = 2**bits, N >> bits
    half = box // 2
    for L in range(3):                    # the layout holds for every L, whether or not the noise check allows it
        K = 1 << L
        for out in ('int', 'bool'):
            tables = rng.randint(0, M, size=(K, M))
            tv = lut.make_test_vector(tables if L else tables[0], bits, L, out).astype(numpy.int64)
            want_of = (lambda f: f << (31 - bits)) if out == 'int' else (lambda f: int(O.MU) if f else -int(O.MU))
            # every mod-switched phase a message can have: [0, N - half) and the wrap [2N - half, 2N) of m = 0
            for b in list(range(0, N - half, K)) + list(range(2 * N - half, 2 * N, K)):
                m = ((b + half) // box) % M if b < N else 0
                for j in range(K):
                    got = _rotate_coef(tv, b, j)
                    assert got == want_of(int(tables[j, m])), (bits, L, out, b, j)


def test_test_vector_per_ciphertext_and_errors():
    tables = numpy.array([[0, 1, 2, 3], [3, 2, 1, 0], [1, 1, 1, 1]])
    tv = lut.make_test_vector(tables, 2, 0)
    assert tv.shape == (3, N)
    for i in range(3):
        assert (tv[i] == lut.make_test_vector(tables[i], 2, 0)).all()
    assert lut.make_test_vector(numpy.zeros((5, 2, 4), int), 2, 1).shape == (5, N)
    with pytest.raises(ValueError):
        lut.make_test_vector([0, 1, 2], 2, 0)
    with pytest.raises(ValueError):
        lut.make_test_vector([0, 1, 2, 3], 2, 3)
    with pytest.raises(ValueError):
        lut.make_test_vector([0, 1, 2, 3], 2, 0, out='float')


def test_modswitch_head_tail_match_the_oracle(emul):
    rng = numpy.random.RandomState(7)
    x = rng.randint(-2**31, 2**31, size=4096, dtype=numpy.int64).astype(numpy.int32)
    x[:8] = [0, -1, 2**31 - 1, -2**31, 2**20, 2**20 - 1, -2**20, 2**21]
    for L in (0, 1, 2):
        want = (O.t32_to_phase(x, (2 * N) >> L).astype(numpy.int64) << L)
        got = numpy.array([emul.emul_modswitch_lut(int(v), L) for v in x])
        assert (got == want).all(), L
        assert (got % (1 << L) == 0).all() and got.min() >= 0 and got.max() < 2 * N
    tv = rng.randint(-2**31, 2**31, size=N, dtype=numpy.int64).astype(numpy.int32)
    for barb in (0, 1, N - 1, N, N + 1, 2 * N - 1):
        got = numpy.empty(N, numpy.int32)
        emul.emul_lut_head(_p(tv), barb, _p(got))
        want = O.shift_torus_polynomial(tv[None, None, :], numpy.array([barb], numpy.int32), invert_powers=True)[0, 0]
        assert (got == want).all(), barb
    acc = rng.randint(-2**31, 2**31, size=(1, 2, N), dtype=numpy.int64).astype(numpy.int32)
    for j in range(4):
        got_a, got_b = numpy.empty(N, numpy.int32), numpy.empty(1, numpy.int32)
        emul.emul_lut_tail(_p(acc), j, _p(got_a), _p(got_b))
        shifted = O.shift_torus_polynomial(acc, numpy.array([(2 * N - j) % (2 * N)], numpy.int32)) if j else acc
        want_a, want_b = O.tlwe_extract_lwe_samples(shifted)
        assert (got_a == want_a[0]).all() and got_b[0] == want_b[0], j


def test_fused_ref_compositions_agree():
    """The oracle compositions the GPU matrix checks against (tests/fused_ref.py) agree with each other at n = 25: the
    LUT composition with the constant test vector mu is the gate bootstrap (also for the rounding ties of the L = 0
    mod-switch), the GLWE composition with zero masks is the LUT composition, the extract2 rows are two gates, and the
    explicit rotation of the gate's initial accumulator is the gate."""
    import fused_ref as F
    keys = O.OracleKeys(G.GATE_SEED, n=25)
    rng = numpy.random.RandomState(8)
    B, n = 12, 25
    x1 = (G.torus32(rng, (B, n)), G.torus32(rng, (B,)))
    x2 = (G.torus32(rng, (B, n)), G.torus32(rng, (B,)))
    x1[1][:4] = [2**20, 2**20 - 1, -2**20, 2**31 - 2**20]            # ties of the rounding, with s1 = 1 and no x2
    c, s1, s2 = 12345678, 1, -3
    gate = F.bootstrap_extract(x1, None, c, s1, s2, O.MU, keys.bk)
    lut0 = F.bootstrap_lut_extract(x1, None, c, s1, s2, numpy.full(N, O.MU, numpy.int32), 0, keys.bk)
    assert (gate[0] == lut0[0]).all() and (gate[1] == lut0[1]).all()
    gate2 = F.bootstrap_extract(x1, x2, c, s1, s2, -2**31, keys.bk)
    lut2 = F.bootstrap_lut_extract(x1, x2, c, s1, s2, numpy.full(N, -2**31, numpy.int32), 0, keys.bk)
    assert (gate2[0] == lut2[0]).all() and (gate2[1] == lut2[1]).all()
    pair = F.bootstrap_extract2((x1, None, c, s1, s2), (x1, x2, c, s1, s2), O.MU, keys.bk)
    assert (pair[0][:B] == gate[0]).all() and (pair[1][B:] == F.bootstrap_extract(x1, x2, c, s1, s2, O.MU, keys.bk)[1]).all()
    tv = G.torus32(rng, (B, N))
    a, b = F.prologue(x1, x2, c, s1, s2)
    glwe = numpy.zeros((B, 2, N), numpy.int32)
    glwe[:, 1] = tv
    want = F.bootstrap_lut_extract((a, b), None, 0, 1, 0, tv, 0, keys.bk)
    got = F.bootstrap_glwe_lut_extract((a, b), glwe, keys.bk)
    assert (got[0] == want[0]).all() and (got[1] == want[1]).all()
    # the gate's initial accumulator (0, X^(2N - barb) mu) rotated explicitly
    barb = O.t32_to_phase(b, 2 * N)
    acc = O.tlwe_noiseless_trivial(O.shift_torus_polynomial(numpy.full((B, 1, N), O.MU, numpy.int32), barb,
                                                            invert_powers=True)[:, 0])
    ea, eb, eacc = F.blind_rotate(acc, O.t32_to_phase(a, 2 * N), keys.bk)
    gate3 = F.bootstrap_extract((a, b), None, 0, 1, 0, O.MU, keys.bk)
    assert (ea == gate3[0]).all() and (eb == gate3[1]).all() and eacc.shape == (B, 2, N)


def test_allowed_table_follows_the_sigma_formula():
    import nufhe_b200
    params = nufhe_b200.NuFHEParameters()
    derived = set()
    for bits in (1, 2, 3):
        for L in range(3):
            for shift in [None] + list(range(bits)):
                if 2.0**-(bits + 2) / lut.lut_sigma(params, L, shift) >= lut.MARGIN_SIGMAS:
                    derived.add((bits, L, shift))
                    lut.check_noise(params, bits, L, shift)
                else:
                    with pytest.raises(ValueError):
                        lut.check_noise(params, bits, L, shift)
    assert derived == lut.ALLOWED
    # the estimates of DESIGN.md section 9
    est = lut._sigma_estimate(params.in_out_params, params.tgsw_params, params.ks_decomp_length,
                              params.ks_log2_base, 0, None)**2
    assert abs(est - (1.28e-5 + 5.0e-6)) < 0.02e-5
    with pytest.raises(ValueError):
        lut.check_noise(params, 2, 0, shift=2)        # shift beyond the message space
    with pytest.raises(ValueError):
        lut.check_noise(params, 4, 0)


class LutFakeEngine(FakeEngine):
    """FakeEngine plus the programmable bootstrap, composed from the oracle's steps like the reference would."""

    def bootstrap_lut_extract(self, x1, x2, c, s1, s2, tv, log2_outputs, bk_int):
        self._count('bootstrap_lut_extract')
        a, b = self._affine(x1, x2, c, s1, s2)
        B, L = b.size, int(log2_outputs)
        K = 1 << L
        barb = (O.t32_to_phase(b.reshape(B), (2 * N) >> L).astype(numpy.int64) << L).astype(numpy.int32)
        bara = (O.t32_to_phase(a.reshape(B, -1), (2 * N) >> L).astype(numpy.int64) << L).astype(numpy.int32)
        tvs = numpy.ascontiguousarray(numpy.broadcast_to(_np(tv).reshape(-1, N), (B, N)))
        acc = O.tlwe_noiseless_trivial(O.shift_torus_polynomial(tvs[:, None, :], barb, invert_powers=True)[:, 0])
        acc = O.blind_rotate(acc, _np(bk_int, True), bara)
        out_a, out_b = numpy.empty((B, K, N), numpy.int32), numpy.empty((B, K), numpy.int32)
        for j in range(K):
            src = O.shift_torus_polynomial(acc, numpy.full(B, 2 * N - j, numpy.int32)) if j else acc
            out_a[:, j], out_b[:, j] = O.tlwe_extract_lwe_samples(src)
        return _t(out_a.reshape(B * K, N)), _t(out_b.reshape(B * K))


@pytest.fixture(scope='module')
def k1():
    import nufhe_b200
    ctx = nufhe_b200.Context(rng=nufhe_b200.DeterministicRNG(G.GATE_SEED), thread=LutFakeEngine())
    sk, ck = ctx.make_key_pair()
    return nufhe_b200, ctx, sk, ck


def test_python_layer_full_adder_fused_and_steps(k1):
    nufhe, ctx, sk, ck = k1
    thr = ctx.thread
    vm_fused = ctx.make_virtual_machine(ck)
    vm_steps = ctx.make_virtual_machine(ck, perf_params=nufhe.PerformanceParameters(ck.params, single_kernel_bootstrap=False))
    a, b, c = numpy.array([1, 0, 1]), numpy.array([1, 1, 0]), numpy.array([1, 0, 0])
    ca, cb, cc = (ctx.encrypt_int(sk, v, 2) for v in (a, b, c))
    assert (ctx.decrypt_int(sk, ca, 2) == a).all()
    adder = vm_fused.make_lut([[v % 2 for v in range(4)], [v // 2 for v in range(4)]], bits=2)
    assert adder.outputs == 2
    results = []
    for vm, counter in ((vm_fused, 'bootstrap_lut_extract'), (vm_steps, 'shift_torus_polynomial')):
        before = thr.calls.get(counter, 0)
        s = vm.int_add(vm.int_add(ca, cb), cc)
        out = vm.lut(adder, s)
        assert thr.calls.get(counter, 0) > before
        total = a + b + c
        assert (ctx.decrypt_int(sk, out[0], 2) == total % 2).all()
        assert (ctx.decrypt_int(sk, out[1], 2) == total // 2).all()
        results.append(out)
    for r_f, r_s in zip(*results):
        assert (r_f.a == r_s.a).all() and (r_f.b == r_s.b).all()


def test_python_layer_bivariate_bool_and_per_ciphertext(k1):
    nufhe, ctx, sk, ck = k1
    vm = ctx.make_virtual_machine(ck)
    x, y = numpy.array([0, 1, 1, 0]), numpy.array([0, 0, 1, 1])
    cx, cy = ctx.encrypt_int(sk, x, 2), ctx.encrypt_int(sk, y, 2)
    # x + y -> bit: x XOR y, as a gate-compatible bit
    t = vm.make_lut([0, 1, 0, 0], bits=2, out='bool')
    r = vm.lut(t, cx, cy)
    assert (ctx.decrypt(sk, r) == (x != y)).all()
    # one table per ciphertext
    tables = numpy.array([[3, 2, 1, 0], [0, 1, 2, 3], [1, 1, 1, 1], [0, 0, 0, 3]])
    t = vm.make_lut(tables, bits=2, log2_outputs=0)
    r = vm.lut(t, cx)
    assert (ctx.decrypt_int(sk, r, 2) == tables[numpy.arange(4), x]).all()
    with pytest.raises(ValueError):
        vm.lut(vm.make_lut(numpy.zeros((4, 8), int), bits=3, log2_outputs=2), cx)   # P = 3, L = 2: not enough margin
    with pytest.raises(ValueError):
        vm.lut(vm.make_lut([0, 1, 2, 3], bits=2), cx, cy, shift=2)
    with pytest.raises(ValueError):
        vm.lut(vm.make_lut([0, 1, 2, 3], bits=2), cx, cy, shift=1)           # measured: 6.6 sigma
    with pytest.raises(ValueError):
        vm.lut(vm.make_lut(list(range(8)), bits=3), ctx.encrypt_int(sk, x, 3))  # measured: 6.7 sigma


def test_python_layer_mask_size_2_steps():
    import nufhe_b200
    ctx = nufhe_b200.Context(rng=nufhe_b200.DeterministicRNG(11), thread=LutFakeEngine())
    sk, ck = ctx.make_key_pair(tlwe_mask_size=2)
    vm = ctx.make_virtual_machine(ck)
    v = numpy.array([0, 1, 2, 3])
    r = vm.lut(vm.make_lut([(3 * m + 1) % 4 for m in range(4)], bits=2), ctx.encrypt_int(sk, v, 2))
    assert (ctx.decrypt_int(sk, r, 2) == (3 * v + 1) % 4).all()
    assert 'bootstrap_lut_extract' not in ctx.thread.calls
