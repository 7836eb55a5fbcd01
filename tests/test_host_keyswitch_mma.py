"""The GEMM formulation of the key switch (tests/ks_mma_ref.py) against the oracle's key switch, on the CPU."""
import numpy

import ks_mma_ref as R
from oracle import oracle as O


def _key(rng, a=None):
    ks_a = rng.randint(-2**31, 2**31, size=(1024, 8, 4, 500), dtype=numpy.int64).astype(numpy.int32)
    ks_b = rng.randint(-2**31, 2**31, size=(1024, 8, 4), dtype=numpy.int64).astype(numpy.int32)
    if a is not None:
        ks_a[:] = a
        ks_b[:] = a
    ks_a[:, :, 0] = 0                   # row d = 0: zero padding in every generated key
    ks_b[:, :, 0] = 0
    return ks_a, ks_b, numpy.zeros((1024, 8, 4), numpy.float32)


def _check(ks, src_a, src_b):
    ra, rb = R.keyswitch(ks[0], ks[1], src_a, src_b)
    wa, wb, _ = O.lwe_keyswitch(*ks, src_a, src_b)
    assert (ra == wa).all() and (rb == wb).all()


def test_k_order_covers_every_row_once():
    j, k, d = R.k_order()
    rows = (j * 8 + k) * 4 + d
    assert j.size == 24576 and numpy.unique(rows).size == 24576 and d.min() == 1


def test_random_inputs():
    rng = numpy.random.RandomState(41)
    ks = _key(rng)
    src_a = rng.randint(-2**31, 2**31, size=(3, 1024), dtype=numpy.int64).astype(numpy.int32)
    src_b = rng.randint(-2**31, 2**31, size=(3,), dtype=numpy.int64).astype(numpy.int32)
    _check(ks, src_a, src_b)


def test_exactness_edge():
    """all digits 3 (8192 one-hot columns per row), key bytes 0xFF and key words -2^31"""
    rng = numpy.random.RandomState(42)
    src_a = numpy.full((2, 1024), -1 - 2**15, numpy.int32)
    assert (R.digits(src_a) == 3).all()
    src_b = numpy.array([0, -2**31], numpy.int32)
    for word in (-1, -2**31):
        _check(_key(rng, word), src_a, src_b)
