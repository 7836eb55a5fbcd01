"""The table and the integer <-> double steps of the FP64 step (csrc/br_phases.cuh), on the host (csrc/host_emul.cpp):
the merged pass-1 twiddle table T[k1][n0] = w^n0 W512^(n0 k1) rounded once from the exact value, the digit built from
the bits of 2^52 + u, and the rounding through the addition of 1.5 2^52 against llrint mod 2^32."""
import ctypes
import os

import mpmath
import numpy
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def emul():
    path = os.path.join(ROOT, 'nufhe_b200', 'csrc', 'libnb_host_emul.so')
    if not os.path.exists(path):
        import __graft_entry__ as g
        g.build()
    lib = ctypes.CDLL(path)
    lib.emul_fft_digit.restype = ctypes.c_double
    lib.emul_fft_digit.argtypes = [ctypes.c_uint]
    lib.emul_fft_rint_lo32.restype = ctypes.c_int
    lib.emul_fft_rint_lo32.argtypes = [ctypes.c_double]
    return lib


def test_pass1_table_is_the_correctly_rounded_product(emul):
    """Every component of T[k1][n0] is within 2^-53 (relative) of the exact e^{2 pi i n0 (1 - 4 k1) / 2048}, as the
    error bound of DESIGN.md section 4 assumes, and the table is stored [k1][n0] (consecutive n0, consecutive
    16-byte elements)."""
    tab = numpy.empty(2 * 512, numpy.float64)
    assert emul.emul_fft_table(tab.ctypes.data_as(ctypes.c_void_p)) == 512
    tab = tab.view(numpy.complex128)
    mpmath.mp.prec = 160
    u = mpmath.mpf(2) ** -53
    for k1 in range(8):
        for n0 in range(64):
            i = emul.emul_fft_tab_t1(k1, n0)
            assert i == k1 * 64 + n0
            a = 2 * mpmath.pi * mpmath.mpf(n0 * (1 - 4 * k1)) / 2048
            for got, exact in ((tab[i].real, mpmath.cos(a)), (tab[i].imag, mpmath.sin(a))):
                assert abs(mpmath.mpf(float(got)) - exact) <= u * abs(exact), (k1, n0, got, exact)


def test_digit_from_bits_is_exact(emul):
    """All 1024 values of u: the double with words 0x43300000 : u, minus 2^52 + 512, is u - 512 exactly."""
    for u in range(1024):
        assert emul.emul_fft_digit(u) == float(u - 512), u


def _llrint_lo32(x):
    r = int(numpy.rint(x))               # round half to even, as llrint in the default rounding mode
    r &= 0xffffffff
    return r - (1 << 32) if r >= 1 << 31 else r


def test_rounding_through_magic_constant_matches_llrint(emul):
    """round(x) mod 2^32 from the low word of x + 1.5 2^52, against llrint mod 2^32: near +-2^45 (the largest
    magnitude the error bound allows), negative values, ties (to even) and +-0.49 around integers."""
    rng = numpy.random.RandomState(20261016)
    base = [0.0, 1.0, -1.0, 2.0**31, -2.0**31, 2.0**32, -2.0**32, 2.0**45, -2.0**45, 2.0**45 - 1, -2.0**45 + 1,
            2.0**50, -2.0**50]
    base += list(rng.randint(-2**45, 2**45, 200).astype(numpy.float64))
    base += list(rng.randint(-2**20, 2**20, 200).astype(numpy.float64))
    xs = []
    for b in base:
        xs += [b, b + 0.49, b - 0.49, b + 0.5, b - 0.5, b + 0.25, b - 0.75]
    xs += list(rng.uniform(-2.0**45, 2.0**45, 2000))
    for x in xs:
        assert emul.emul_fft_rint_lo32(x) == _llrint_lo32(x), x
