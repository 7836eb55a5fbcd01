"""The FP64 step of the throughput shape (csrc/kernels.cuh: br_fft_step) at kernel level, against the CPU oracle: plain
external products and explicit blind rotations in both throughput shapes (FP64 and NTT step), keys and accumulators at
the extreme magnitudes of the FP64 error bound (DESIGN.md section 3), the device key spectra against the host's, the
integrality check at the edges of the 32-bit range, and which prepared key rows a launch runs the FP64 step on.

"Spoiling" a prepared key zeroes the FP64 part of its rows after preparation.  The FP64 step then multiplies by the
zero polynomial: a plain product gives 0 and a CMux step leaves the accumulator as it was.  The NTT step does not read
that part and gives the right bits.  That shows which step ran."""
import ctypes
import os

import numpy
import pytest
import torch

import gen_inputs as G
from oracle import oracle as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FFT_U64 = 16 * 512 * 2            # the FP64 part at the end of every engine key row (br_phases.cuh: BK_FFT_U64)
# the throughput shape at every batch: no pair, wide2 or wide launches
THROUGHPUT = {'NUFHE_B200_WIDE_MAX': '0', 'NUFHE_B200_WIDE2_MAX': '0', 'NUFHE_B200_PAIR_MAX': '0'}
EDGE_ROTATIONS = numpy.array([0, 1, 1023, 1024, 1025, 2047], numpy.int32)
DIG_MIN, DIG_MAX = 0x7FE00000, 0x7FDFF000        # accumulator coefficients whose two digits are both -512 / both +511


@pytest.fixture(scope='module')
def keys():
    return O.OracleKeys(G.GATE_SEED)


@pytest.fixture(scope='module')
def slots():
    """resident CTAs of a throughput-shape launch (2 per SM, 2 ciphertexts each): a wave is 2 * slots ciphertexts"""
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count * 2


@pytest.fixture(scope='module')
def emul():
    path = os.path.join(ROOT, 'nufhe_b200', 'csrc', 'libnb_host_emul.so')
    if not os.path.exists(path):
        import __graft_entry__ as g
        g.build()
    return ctypes.CDLL(path)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _engine(monkeypatch, fft, env=THROUGHPUT):
    """A fresh engine (the knobs are read when its context is created) with the FP64 step ('1') or the NTT step ('0')
    for keys that have spectra; env=None keeps the default shape thresholds."""
    from nufhe_b200.engine import Engine
    for k in list(THROUGHPUT) + ['NUFHE_B200_FORCE_CHUNKS']:
        monkeypatch.delenv(k, raising=False)
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    monkeypatch.setenv('NUFHE_B200_FFT', fft)
    return Engine()


def _prepare(eng, bk, spoil=False):
    bk_int = eng.bk_prepare(eng.to_device(bk))
    if spoil:
        bk_int[:, -FFT_U64:] = 0
    return bk_int


def _external(eng, bk_int, acc, row):
    return eng.to_host(eng.external_product(eng.to_device(acc), bk_int, row))


def _rotate(eng, bk_int, acc, bara, extract=False):
    out_a, out_b, acc_out = eng.blind_rotate(eng.to_device(acc), eng.to_device(bara), bk_int, extract=extract,
                                             return_accum=True)
    if extract:
        return eng.to_host(acc_out), eng.to_host(out_a), eng.to_host(out_b)
    return eng.to_host(acc_out)


def _extreme_key():
    """Six key rows (reference form) whose eight polynomials all carry one extreme pattern of the host tests
    (tests/test_host_fft.py): -2^31, -2^31 + 2^15, 2^31 - 1, the two alternations of -2^31 and 2^31 - 1, and the
    sign pattern aligned with the negacyclic wrap of output coefficient 0."""
    n = numpy.arange(1024)
    s = numpy.where(n == 0, 1, -1)
    patterns = [numpy.full(1024, -2**31), numpy.full(1024, -2**31 + 2**15), numpy.full(1024, 2**31 - 1),
                numpy.where(n % 2 == 0, -2**31, 2**31 - 1), numpy.where(n % 2 == 0, 2**31 - 1, -2**31),
                s[(-n) % 1024] * -(2**31 - 2**16) - 2**15]
    raw = numpy.stack([numpy.broadcast_to(numpy.asarray(p, numpy.int64), (2, 2, 2, 1024)) for p in patterns])
    assert raw.min() >= -2**31 and raw.max() < 2**31
    return O.bk_transform(raw.astype(numpy.int32))


def _digit_patterns():
    """sign patterns (True = -512, False = +511) of both digits: all -512, all +511, alternating (aligned with the
    alternating keys), and alternating reversed"""
    n = numpy.arange(1024)
    return numpy.stack([numpy.ones(1024, bool), numpy.zeros(1024, bool), n % 2 == 0, n[::-1] % 2 != 0])


def _with_coefficient(raw, where, value):
    """reference form of the raw key with raw[where] = value, which may lie outside int32: the transform is linear
    over the field, so the key is the sum of two transforms"""
    base, one = raw.copy(), numpy.zeros_like(raw)
    step = 1 if value > 0 else -1
    base[where], one[where] = value - step, step
    return O.ff_add(O.bk_transform(base), O.bk_transform(one))


# ---- T1: the plain external product (ACCUMULATE = false in the last phase) -------------------------------------------

def test_plain_external_product_in_both_throughput_shapes(monkeypatch, keys, slots):
    """nb_external_product (tgsw_transformed_external_mul) in the throughput shape, with the FP64 and the NTT step:
    batches 1, 2, an odd batch (its last slot replays a ciphertext) and one chain more than a wave (the persistent
    queue); the first, second and last key rows; bit for bit against the oracle."""
    rng = G.rs(601)
    rows = (0, 1, keys.bk.shape[0] - 1)
    accs = {B: G.torus32(rng, (B, 2, 1024)) for B in (1, 2, 3, 2 * slots + 1)}
    want = {(B, r): O.tgsw_external_mul(acc, keys.bk, r) for B, acc in accs.items() for r in rows}
    for fft in ('1', '0'):
        eng = _engine(monkeypatch, fft)
        bk_int, spoiled = _prepare(eng, keys.bk), _prepare(eng, keys.bk, spoil=True)
        for B, acc in accs.items():
            for r in rows:
                assert (_external(eng, bk_int, acc, r) == want[B, r]).all(), (fft, B, r)
                got = _external(eng, spoiled, acc, r)
                if fft == '1':
                    assert (got == 0).all(), (B, r)
                else:
                    assert (got == want[B, r]).all(), (B, r)


def test_plain_external_product_at_default_thresholds(monkeypatch, keys):
    """2000 ciphertexts with the default shape thresholds take the FP64 throughput shape"""
    rng = G.rs(602)
    acc = G.torus32(rng, (2000, 2, 1024))
    eng = _engine(monkeypatch, '1', env=None)
    bk_int, spoiled = _prepare(eng, keys.bk), _prepare(eng, keys.bk, spoil=True)
    for r in (0, keys.bk.shape[0] - 1):
        want = O.tgsw_external_mul(acc, keys.bk, r)
        assert (_external(eng, bk_int, acc, r) == want).all(), r
        assert (_external(eng, spoiled, acc, r) == 0).all(), r


# ---- T2: explicit blind rotation (accumulator and rotation amounts given) -------------------------------------------

@pytest.mark.parametrize('n', [1, 7, 25])
def test_explicit_blind_rotation_in_both_throughput_shapes(monkeypatch, keys, slots, n):
    """nb_blind_rotate with the first n rows of the gate key: the final accumulator and the extracted sample equal the
    oracle's, with the FP64 and the NTT step, for a ragged batch and one with more chains than a wave (time-sliced).
    At n = 25 the FP64 shape also runs with 3 forced chunks: they start at steps 0, 9 and 18, so a chunk resumes on an
    odd step (the rotation amounts' double buffer) from accumulators parked by another CTA."""
    rng = G.rs(610 + n)
    bk = keys.bk[:n]
    for B in (3, 2 * slots + 3):
        acc = G.torus32(rng, (B, 2, 1024))
        bara = G.torus32(rng, (B, n), 0, 2048)
        m = min(bara.size, 3 * EDGE_ROTATIONS.size)
        bara.reshape(-1)[:m] = numpy.resize(EDGE_ROTATIONS, m)
        bara.reshape(-1)[-m:] = numpy.resize(EDGE_ROTATIONS[::-1], m)
        want = O.blind_rotate(acc, bk, bara)
        want_a, want_b = O.tlwe_extract_lwe_samples(want)
        runs = [('1', THROUGHPUT), ('0', THROUGHPUT)]
        if n == 25 and B > 3:
            runs.append(('1', dict(THROUGHPUT, NUFHE_B200_FORCE_CHUNKS='3')))
        for fft, env in runs:
            eng = _engine(monkeypatch, fft, env)
            bk_int = _prepare(eng, bk)
            got, got_a, got_b = _rotate(eng, bk_int, acc, bara, extract=True)
            assert (got == want).all(), (B, fft, env)
            assert (got_a == want_a).all() and (got_b == want_b).all(), (B, fft, env)
            bk_int[:, -FFT_U64:] = 0
            got = _rotate(eng, bk_int, acc, bara)
            if fft == '1':
                assert (got == acc).all(), (B, env)
            else:
                assert (got == want).all(), B


# ---- T3: extreme magnitudes through the device kernel ---------------------------------------------------------------

def test_extreme_keys_and_digits_through_the_fp64_step(monkeypatch, emul):
    """Keys at the ends of the 32-bit range and digits at -512 / +511, with signs aligned to the keys: the products
    reach the largest magnitudes of the error bound.  The FP64 step must give the oracle's bits, and so must the host
    execution of the same passes (emul_fft_step).  Plain products, and CMux steps by X^1024 from accumulators of
    0xC0100000 / 0xC0100800, whose difference rot(acc) - acc = -2 acc = 0x7FE00000 / 0x7FDFF000 has all digits at
    -512 / +511.  (With the key at -2^31 everywhere every product is 0 mod 2^32; the FP64 step still has to compute
    its high half, -2^15 times the digit sums, exactly.)"""
    xbk = _extreme_key()
    neg = _digit_patterns()
    plain = numpy.repeat(numpy.where(neg, DIG_MIN, DIG_MAX).astype(numpy.int32)[:, None, :], 2, axis=1)
    cmux = numpy.repeat(numpy.where(neg, 0xC0100000, 0xC0100800).astype(numpy.uint32).view(numpy.int32)[:, None, :],
                        2, axis=1)
    digits = numpy.repeat(numpy.where(neg, -512, 511)[:, None, None, :], 2, axis=1)
    digits = numpy.repeat(digits, 2, axis=2)                       # (B, mi, j, N)
    assert (O.tgsw_decompose(plain) == digits).all()
    diff = (numpy.uint32(0) - 2 * cmux.view(numpy.uint32)).view(numpy.int32)
    assert (O.tgsw_decompose(diff) == digits).all()
    B = plain.shape[0]
    bara = numpy.full((B, 1), 1024, numpy.int32)
    eng = _engine(monkeypatch, '1')
    bk_int, spoiled = _prepare(eng, xbk), _prepare(eng, xbk, spoil=True)
    for r in range(xbk.shape[0]):
        want = O.tgsw_external_mul(plain, xbk, r)
        assert (_external(eng, bk_int, plain, r) == want).all(), r
        assert (_external(eng, spoiled, plain, r) == 0).all(), r
        want_cmux = O.blind_rotate(cmux, xbk[r:r + 1], bara)
        assert (_rotate(eng, bk_int[r:r + 1], cmux, bara) == want_cmux).all(), r
        assert (_rotate(eng, spoiled[r:r + 1], cmux, bara) == cmux).all(), r
        row = numpy.ascontiguousarray(xbk[r])
        for c in range(0, B, 2):
            host = plain[c:c + 2].copy()
            assert emul.emul_fft_step(_p(host), _p(row), None, ctypes.c_int(2)) == 0
            assert (host == want[c:c + 2]).all(), (r, c)
            host = cmux[c:c + 2].copy()
            rot = numpy.full(2, 1024, numpy.int32)
            assert emul.emul_fft_step(_p(host), _p(row), _p(rot), ctypes.c_int(2)) == 0
            assert (host == want_cmux[c:c + 2]).all(), (r, c)


# ---- T4: the key spectra nb_bk_prepare writes -----------------------------------------------------------------------

def test_device_key_spectra_equal_the_host_spectra(monkeypatch, keys, emul):
    """The FP64 part of each prepared row (bk_spectra_kernel) equals, bit for bit, the host computation of the same
    passes (emul_fft_key_row) -- for gate-key rows spread over the key and for the extreme keys."""
    eng = _engine(monkeypatch, '1')
    host = numpy.empty(FFT_U64, numpy.float64)
    for bk, rows in ((keys.bk, [0, 1, 37, 250, 498, 499]), (_extreme_key(), list(range(6)))):
        dev = eng.to_host(eng.bk_prepare(eng.to_device(bk))[rows, -FFT_U64:], True)
        for i, r in enumerate(rows):
            assert emul.emul_fft_key_row(_p(numpy.ascontiguousarray(bk[r])), _p(host)) == 0
            assert (dev[i] == host.view(numpy.uint64)).all(), r


# ---- T5: the integrality check at its edges -------------------------------------------------------------------------

@pytest.mark.parametrize('where', [(2, 1, 1, 1, 1023), (0, 0, 0, 0, 0)], ids=['last_row_m7_c1023', 'row0_m0_c0'])
@pytest.mark.parametrize('value', [2**31, -2**31 - 1], ids=['2^31', '-2^31-1'])
def test_one_coefficient_outside_int32_keeps_the_ntt_step(monkeypatch, keys, where, value):
    """A key whose only coefficient outside [-2^31, 2^31) sits at the last position of the last polynomial of the last
    row, or at the first position of the first one, has no usable spectra: the throughput shape keeps the NTT step
    (spoiling changes nothing) and gives the oracle's bits."""
    rng = G.rs(620)
    bk = _with_coefficient(keys.bk_raw[:3], where, value)
    acc = G.torus32(rng, (3, 2, 1024))
    bara = G.torus32(rng, (3, 3), 0, 2048)
    want = O.blind_rotate(acc, bk, bara)
    eng = _engine(monkeypatch, '1')
    for spoil in (False, True):
        assert (_rotate(eng, _prepare(eng, bk, spoil), acc, bara) == want).all(), spoil


def test_extreme_int32_coefficients_take_the_fp64_step(monkeypatch):
    """-2^31 and 2^31 - 1 everywhere are integral: the FP64 step runs (on the spoiled key it leaves the accumulator
    as it was) and gives the oracle's bits"""
    rng = G.rs(621)
    bk = _extreme_key()[[0, 2]]
    acc = G.torus32(rng, (3, 2, 1024))
    bara = G.torus32(rng, (3, 2), 1, 2048)
    want = O.blind_rotate(acc, bk, bara)
    eng = _engine(monkeypatch, '1')
    assert (_rotate(eng, _prepare(eng, bk), acc, bara) == want).all()
    assert (_rotate(eng, _prepare(eng, bk, spoil=True), acc, bara) == acc).all()


# ---- T6: which rows of a prepared buffer the FP64 step may read ---------------------------------------------------

def test_fp64_step_only_on_rows_of_one_integral_preparation(monkeypatch, keys):
    """nb_bk_prepare records, per call, whether the key it prepared has spectra.  A launch may take the FP64 step only
    if every row it reads comes from one such call: (a) a buffer whose first half holds an integral key and whose
    second half was then prepared from a random-field key (no spectra), (b) an integral key overwritten by a
    random-field key, (c) the reverse, (d) a plain product on the last row of a registered key.  All equal the
    oracle; spoiling shows which step ran."""
    from nufhe_b200.engine import _ptr
    rng = G.rs(630)
    n, B = 8, 3
    field = G.ff_numbers(rng, (n, 2, 2, 2, 1024))
    gate = keys.bk[:n]
    acc = G.torus32(rng, (B, 2, 1024))
    bara = G.torus32(rng, (B, n), 1, 2048)
    eng = _engine(monkeypatch, '1')
    row_u64 = eng.lib.nb_bk_row_u64()

    def buffer(*parts):
        """one buffer of n rows, prepared by one nb_bk_prepare call per (first row, reference rows)"""
        buf = eng.empty((n, row_u64), torch.int64)
        for first, src in parts:
            eng._call('nb_bk_prepare', _ptr(eng.to_device(src)), _ptr(buf[first:first + src.shape[0]]), src.shape[0])
        return buf

    def spoil(buf):
        buf[:, -FFT_U64:] = 0            # in place: the key stays where it was registered

    # (a) integral rows [0, n/2), then random-field rows [n/2, n) into the same buffer
    h = n // 2
    buf = buffer((0, gate[:h]), (h, field[h:]))
    want = O.blind_rotate(acc, numpy.concatenate([gate[:h], field[h:]]), bara)
    want_half = O.blind_rotate(acc, gate[:h], bara[:, :h])
    assert (_rotate(eng, buf, acc, bara) == want).all()
    assert (_rotate(eng, buf[:h], acc, bara[:, :h]) == want_half).all()
    spoil(buf)
    assert (_rotate(eng, buf, acc, bara) == want).all()                     # the NTT step
    assert (_rotate(eng, buf[:h], acc, bara[:, :h]) == acc).all()            # the FP64 step on the integral rows
    # (b) an integral key, then a random-field key over it
    buf = buffer((0, gate), (0, field))
    want = O.blind_rotate(acc, field, bara)
    assert (_rotate(eng, buf, acc, bara) == want).all()
    spoil(buf)
    assert (_rotate(eng, buf, acc, bara) == want).all()
    # (c) a random-field key, then an integral key over it; (d) a plain product on its last row
    buf = buffer((0, field), (0, gate))
    want = O.blind_rotate(acc, gate, bara)
    want_last = O.tgsw_external_mul(acc, gate, n - 1)
    assert (_rotate(eng, buf, acc, bara) == want).all()
    assert (_external(eng, buf, acc, n - 1) == want_last).all()
    spoil(buf)
    assert (_rotate(eng, buf, acc, bara) == acc).all()
    assert (_external(eng, buf, acc, n - 1) == 0).all()
