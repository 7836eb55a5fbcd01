"""The FP64 step of the throughput shape (csrc/br_phases.cuh: FP64 step) executed on the host (csrc/host_emul.cpp):
its transform chain must round to the exact negacyclic products, with a wide margin, on adversarial inputs, and one
whole CMux step must give the oracle's bits."""
import ctypes
import os

import numpy
import pytest

import gen_inputs as G
from oracle import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def emul():
    path = os.path.join(ROOT, 'nufhe_b200', 'csrc', 'libnb_host_emul.so')
    if not os.path.exists(path):
        import __graft_entry__ as g
        g.build()
    return ctypes.CDLL(path)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _negacyclic(a, b):
    """exact a * b mod X^1024 + 1 for int64 inputs (products and sums stay below 2^63 here)"""
    n = a.shape[-1]
    full = numpy.zeros(2 * n, dtype=object)
    a, b = [int(x) for x in a], [int(x) for x in b]
    for i, x in enumerate(a):
        if x:
            for j, y in enumerate(b):
                full[i + j] += x * y
    return numpy.array([full[k] - full[k + n] for k in range(n)], dtype=object)


def _negacyclic_fast(a, b):
    """the same through an integer circulant: a (n,) int64, b (n,) int64, exact in int64 for |a| <= 2^10, |b| <= 2^16"""
    n = a.shape[0]
    idx = (numpy.arange(n)[:, None] - numpy.arange(n)[None, :])
    sign = numpy.where(idx < 0, -1, 1).astype(numpy.int64)
    m = b[idx % n] * sign            # m[k, j] = +-b[k - j]
    return m @ a


def _halves(k):
    lo = ((k + 2**15) & 0xffff) - 2**15
    return lo, (k - lo) // 2**16


def _check_product(emul, dig, key):
    """dig (4, 1024) signed digits, key (4, 1024) centred 32-bit: returns the largest distance of the unrounded FP64
    result from the exact integer products of both key halves"""
    out = numpy.empty((2, 1024), numpy.float64)
    emul.emul_fft_product(_p(numpy.ascontiguousarray(dig, numpy.float64)), _p(numpy.ascontiguousarray(key, numpy.int64)), _p(out))
    lo, hi = _halves(key.astype(numpy.int64))
    err = 0.0
    for h, part in enumerate((lo, hi)):
        exact = sum(_negacyclic_fast(dig[d].astype(numpy.int64), part[d]) for d in range(4))
        assert numpy.abs(exact).max() < 2**53
        err = max(err, float(numpy.abs(out[h] - exact.astype(numpy.float64)).max()))
        assert (numpy.rint(out[h]).astype(numpy.int64) == exact).all()
    return err


def test_negacyclic_helper():
    rng = numpy.random.RandomState(1)
    a = rng.randint(-512, 512, 1024).astype(numpy.int64)
    b = rng.randint(-2**15, 2**15, 1024).astype(numpy.int64)
    assert (_negacyclic_fast(a, b) == _negacyclic(a, b).astype(numpy.int64)).all()


def test_fft_product_is_exact_on_adversarial_inputs(emul):
    """The DESIGN.md section 3 bound says the rounding error stays below 0.5; these inputs push the products to their
    extreme magnitudes: all digits -512 (or +-512 aligned with the key signs) and key halves at +-2^15, alternating
    patterns, and random inputs.  Every result rounds to the exact integer, with an error far below 0.5."""
    worst = 0.0
    n = numpy.arange(1024)
    cases = []
    # aligned extremes: digits at -512 / 511 everywhere, keys at -2^31 (lo = 0, hi = -2^15), at
    # -2^31 + 2^15 (lo = -2^15, hi = -2^15 + 1) and at 2^31 - 1
    cases.append((numpy.full((4, 1024), -512), numpy.full((4, 1024), -2**31)))
    cases.append((numpy.full((4, 1024), -512), numpy.full((4, 1024), -2**31 + 2**15)))
    cases.append((numpy.full((4, 1024), 511), numpy.full((4, 1024), 2**31 - 1)))
    # alternating signs (the negacyclic product of a with its own sign pattern reversed maximises one coefficient)
    alt = numpy.where(n % 2 == 0, -512, 511)
    cases.append((numpy.stack([alt] * 4), numpy.stack([numpy.where(n % 2 == 0, -2**31, 2**31 - 1)] * 4)))
    rev = numpy.where(n[::-1] % 2 == 0, 1, -1)
    cases.append((numpy.stack([numpy.where(rev > 0, 511, -512)] * 4), numpy.stack([numpy.where(n % 2 == 0, 2**31 - 1, -2**31)] * 4)))
    # sign pattern aligned with the negacyclic wrap for output coefficient 0: c_0 = sum a_j b_{-j}, b_{-j} = -b_{1024-j}
    s = numpy.where(n == 0, 1, -1)
    cases.append((numpy.stack([numpy.full(1024, -512)] * 4), numpy.stack([(s[(-n) % 1024] * -(2**31 - 2**16) - 2**15)] * 4)))
    rng = numpy.random.RandomState(20261015)
    for _ in range(6):
        cases.append((rng.randint(-512, 512, (4, 1024)), rng.randint(-2**31, 2**31, (4, 1024), dtype=numpy.int64)))
        cases.append((rng.choice([-512, 511], (4, 1024)), rng.choice([-2**31, 2**31 - 1, -2**31 + 2**15, 2**31 - 2**15 - 1], (4, 1024))))
    for dig, key in cases:
        worst = max(worst, _check_product(emul, numpy.asarray(dig), numpy.asarray(key, numpy.int64)))
    assert worst < 2**-6, worst


def test_fft_step_matches_oracle(emul):
    """One CMux step and one plain external product of the FP64 step (csrc/br_phases.cuh) on the host, with a key made
    by the oracle's key generation (integral coefficients), against the oracle; edge rotation amounts."""
    keys = O.OracleKeys(20260923)
    rng = G.rs(79)
    for nct in (1, 2):
        for rots in ([0, 1024], [1023, 2047], [5, 77]):
            acc = G.torus32(rng, (nct, 2, 1024))
            rot = numpy.array(rots[:nct], numpy.int32)
            a = acc.copy()
            assert emul.emul_fft_step(_p(a), _p(keys.bk[3]), _p(rot), ctypes.c_int(nct)) == 0
            assert (a == O.blind_rotate(acc, keys.bk[3:4], rot.reshape(nct, 1))).all()
        a = acc.copy()
        assert emul.emul_fft_step(_p(a), _p(keys.bk[1]), None, ctypes.c_int(nct)) == 0
        assert (a == O.tgsw_external_mul(acc, keys.bk, 1)).all()


def test_fft_key_row_accepts_exactly_the_32_bit_range(emul):
    """Key preparation on the host (emul_fft_key_row, the computation of kernels.cuh: bk_spectra_kernel): the extreme
    centred 32-bit coefficients -2^31 and 2^31 - 1 are accepted; one coefficient just outside that range, at the last
    position of the last polynomial of the row, rejects the whole row."""
    out = numpy.empty(16 * 512 * 2, numpy.float64)
    lows = numpy.full((2, 2, 2, 1024), -2**31, numpy.int32)
    assert emul.emul_fft_key_row(_p(O.bk_transform(lows)), _p(out)) == 0
    spec = out.view(numpy.complex128).reshape(8, 2, 512)        # [m][h][P]
    assert (spec[:, 0] == 0).all()                 # -2^31 = 0 + 2^16 * (-2^15): the low half is zero ...
    assert (numpy.abs(spec[:, 1]) > 0).all()       # ... the high half, all -2^15, is 2 c / (1 - z) at each root z
    highs = numpy.full((2, 2, 2, 1024), 2**31 - 1, numpy.int32)
    assert emul.emul_fft_key_row(_p(O.bk_transform(highs)), _p(out)) == 0
    for edge, step in ((2**31 - 1, 1), (-2**31, -1)):          # 2^31, -2^31 - 1 at (m = 7, coefficient 1023)
        raw = numpy.zeros((2, 2, 2, 1024), numpy.int32)
        one = numpy.zeros_like(raw)
        raw[1, 1, 1, 1023], one[1, 1, 1, 1023] = edge, step
        assert emul.emul_fft_key_row(_p(O.ff_add(O.bk_transform(raw), O.bk_transform(one))), _p(out)) == -1
        assert emul.emul_fft_key_row(_p(O.bk_transform(raw)), _p(out)) == 0


def test_fft_step_refuses_random_field_keys(emul):
    """A key whose polynomials are not centred 32-bit integers (uniformly random field elements) has no spectra: such
    keys keep the NTT step in every shape."""
    rng = G.rs(80)
    bk = G.ff_numbers(rng, (2, 2, 2, 1024))
    acc = G.torus32(rng, (1, 2, 1024))
    assert emul.emul_fft_step(_p(acc), _p(bk), None, ctypes.c_int(1)) == -1
