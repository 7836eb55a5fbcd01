"""The host model of the key switch's launch shapes, variance sum and edge inputs (tests/ks_ref.py), on the CPU."""
import numpy

import ks_mma_ref as R
import ks_ref as K
from oracle import oracle as O

GATHER_132 = {128, 66, 44, 33, 26, 22, 18, 16, 14, 13, 12, 11, 10, 9, 8, 7, 6, 5, 4, 3, 2, 1}
GATHER_114 = {114, 57, 38, 28, 22, 19, 16, 14, 12, 11, 10, 9, 8, 7, 6, 5, 4, 3, 2, 1}


def test_split_sets():
    assert set(K.gather_bands(132)) == GATHER_132
    assert set(K.gather_bands(114)) == GATHER_114
    assert set(K.mma_bands(132)) == {8, 4, 2, 1}
    assert set(K.mma_bands(114)) == {4, 2, 1}
    # K is halved from 8 to 16 slices only while 16 tiles x 8 slices leave half of the SMs idle: 256 SMs or more
    assert K.mma_launch(1, 255)[2] == 8 and K.mma_launch(1, 256)[2] == 16


def test_band_edges_132():
    assert K.mma_batches(132) == {8: [1, 256], 4: [257, 512], 2: [513, 1024], 1: [1025]}
    g = K.gather_batches(132)
    assert g[128] == [1, 32] and g[66] == [33, 64] and g[44] == [65, 96] and g[1] == [2113, 2144]
    for sm in (132, 114):
        for s, bs in K.gather_batches(sm).items():
            for B in bs:
                assert K.gather_launch(B, sm)[2] == s
            lo = bs[0]
            if lo > 1:                               # one batch less is in the band with more splits
                assert K.gather_launch(lo - 1, sm)[2] > s
        for s, bs in K.mma_batches(sm).items():
            assert all(K.mma_launch(B, sm)[2] == s for B in bs)
            if bs[0] > 1:
                assert K.mma_launch(bs[0] - 1, sm)[2] > s
    bs = K.matrix_batches(132)
    assert {1, 256, 257, 512, 513, 1024, 1025, 4097, 16384} <= set(bs)


def test_j_slices():
    """every split gives slices of whole variance blocks that cover j exactly once, including j_per that does not
    divide 1024 (44 and 26 splits)"""
    assert K.gather_launch(65, 132)[2:] == (44, 24)
    assert K.gather_launch(129, 132)[2:] == (26, 40)
    for s in range(1, 129):
        sl = K.j_slices(s)
        assert len(sl) == s and sl[0][0] == 0 and sl[-1][1] == 1024
        assert all(b % K.CV_BLOCK_J == 0 and e % K.CV_BLOCK_J == 0 and b <= e for b, e in sl)
        assert all(sl[i][1] == sl[i + 1][0] for i in range(s - 1))


def _cv(rng):
    return rng.uniform(0.0, 1e-6, size=(1024, 8, 4)).astype(numpy.float32)


def test_variance_restatement():
    """equals the oracle's running float32 sum to float32 rounding, and the float64 sum within the bound of its 190
    additions on any path: |error| <= 190 * 2^-24 * sum |terms|"""
    rng = numpy.random.RandomState(51)
    ks_cv = _cv(rng)
    src = K.edge_rows(rng, 40)
    got = K.variance(ks_cv, src)
    assert got.dtype == numpy.float32 and got.shape == (40,)
    zeros = numpy.zeros((1024, 8, 4, 1), numpy.int32)
    _, _, want = O.lwe_keyswitch(zeros, numpy.zeros((1024, 8, 4), numpy.int32), ks_cv, src,
                                 numpy.zeros(40, numpy.int32))
    assert numpy.allclose(got, want, rtol=2e-5, atol=0)
    exact, mag = K.variance_f64(ks_cv, src)
    assert K.VARIANCE_ADDS == 190
    assert (numpy.abs(got.astype(numpy.float64) - exact) <= K.VARIANCE_ADDS * 2.0**-24 * mag).all()
    # the block shape is not the running sum: somewhere the two differ in the last bits
    assert not (got.view(numpy.uint32) == want.view(numpy.uint32)).all()


def test_variance_terms():
    """a one-hot ks_cv picks exactly the digits the inputs claim"""
    src = K.edge_rows(numpy.random.RandomState(52), 3)
    ks_cv = numpy.zeros((1024, 8, 4), numpy.float32)
    ks_cv[:, :, 3] = 1.0
    assert K.variance(ks_cv, src)[0] == 8192 and K.variance(ks_cv, src)[1] == 0


def test_edge_coefficients_have_their_digits():
    edges = K.edge_coefficients()
    coeffs = K.i32(numpy.array([c for c, _ in edges]))
    want = numpy.array([d for _, d in edges])
    assert (R.digits(coeffs[None])[0] == want).all()
    # each digit value 1..3 alone in each of the 8 positions, at both rounding edges
    single = [(tuple(d)) for _, d in edges if sum(x != 0 for x in d) == 1]
    assert len(single) == 2 * 3 * 8 and len(set(single)) == 3 * 8
    # one below the lowest and one above the highest coefficient that rounds to a word round to another word
    for c, d in edges[4:]:
        step = -1 if (c & 0xFFFF) == 0x8000 else 1
        assert (R.digits(K.i32([[c + step]]))[0, 0] != numpy.array(d)).any()


def test_edge_rows():
    rng = numpy.random.RandomState(53)
    src = K.edge_rows(rng, 60)
    d = R.digits(src)
    assert (d[0] == 3).all() and (d[1] == 0).all()
    assert src[1].view(numpy.uint32).min() == K.ALL_ZERO_WRAP
    n_edges = len(K.edge_coefficients())
    assert set(src[2].view(numpy.uint32)[:n_edges].tolist()) == {c for c, _ in K.edge_coefficients()}
    assert (src[3] == numpy.roll(src[2], 1)).all()


def test_fold_pairs_wrap():
    rng = numpy.random.RandomState(54)
    target = K.edge_rows(rng, 8)
    target[7, :2] = [-1, 0]                             # 2^32 - 1 has no wrapping pair; 0 has
    s1, s2 = K.fold_pair(rng, target)
    total = K.u32(s1) + K.u32(s2)
    assert ((total & 0xFFFFFFFF) == K.u32(target)).all()
    assert ((total >= 2**32) == (K.u32(target) != 0xFFFFFFFF)).all()
    with numpy.errstate(over='ignore'):
        folded = (s1 + s2).astype(numpy.int32)
    assert (R.digits(folded) == R.digits(target)).all()


def test_tagged_key():
    ks_a, ks_b, ks_cv = K.tagged_key(in_size=4, t=2, base=4, n=5)
    assert ks_a.shape == (4, 2, 4, 5) and ks_b.shape == (4, 2, 4) and ks_cv.shape == (4, 2, 4)
    assert (ks_a[:, :, 0] == 0).all() and (ks_b[:, :, 0] == 0).all()
    words = numpy.concatenate([ks_a[:, :, 1:].ravel(), ks_b[:, :, 1:].ravel()])
    assert numpy.unique(words).size == words.size
    assert (ks_a.view(numpy.uint32) >> 24).max() > 0      # the high byte is used too


def test_edge_keys():
    rng = numpy.random.RandomState(55)
    for kind in ('random', 'bytes_ff', 'min_word'):
        ks_a, ks_b, _ = K.edge_key(kind, rng)
        assert (ks_a[:, :, 0] == 0).all() and (ks_b[:, :, 0] == 0).all()
    ks_a, ks_b, _ = K.edge_key('bytes_ff', rng)
    assert (ks_a[:, :, 1:] == -1).all() and (ks_b[:, :, 1:] == -1).all()
    ks_a, _, _ = K.edge_key('pad', rng)
    assert (ks_a[:, :, 0] != 0).any()
