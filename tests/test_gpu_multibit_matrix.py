"""Multi-bit bootstrap keys (DESIGN.md section 14) in every schedule, bit for bit against the C oracle's exact multi-bit
rotation (O.blind_rotate_mb, composed with the oracle's head and tail steps by tests/multibit_ref.py).

A multi-bit key always runs the FP64 throughput shape (2 ciphertexts per CTA), so one wave W is 4 x SMs ciphertexts.
Schedules: the default; no start-up stagger (single waves); one chunk per chain (multi-wave launches); forced chunks
that resume chains on odd groups and end with a one-group chunk (n = 26: 5 chunks at groups 0, 3, 6, 9, 12; n = 500: 4
chunks at 0, 63, 126, 189); and the wide, wide2 and pair thresholds forced, which a multi-bit key must ignore.

Every call goes through the C ABI with its outputs inside guard rows that must keep their sentinel.  The first rows of
every input set are built so that every ordered pair of targets is some group's (abar_2g, abar_2g+1): for the gate
targets these are the rotation edges 0, 1, 1023, 1024, 1025, 2047 at the centre and at the rounding tie (pairs whose sum
wraps past 2N included), for the LUT modes the rounding ties of the LUT mod-switch.  Separately, keys, test vectors and
rotations at the extremes of the kernel's exactness bound run at n = 2 and 8, and the C ABI's refusals and key
re-registration are checked.

The oracle runs once per mode and dimension on the largest batch any cell uses; every cell compares its prefix."""
import functools
import types

import numpy
import pytest
import torch

import fused_ref as F
import gen_inputs as G
import multibit_ref as M
from fused_ref import gate_mode, glwe_mode, lut_mode, ptr, x2_mode
from nufhe_b200 import _native
from oracle import oracle as O

pytestmark = pytest.mark.gpu
N = 1024
SEED = 20261017

# the multi-bit compositions on the exact oracle, with fused_ref's signatures (bk: the key's transformed rows)
EXACT = types.SimpleNamespace(
    bootstrap_extract=functools.partial(M.bootstrap_extract, rotate=M.blind_rotate_oracle),
    bootstrap_lut_extract=functools.partial(M.bootstrap_lut_extract, rotate=M.blind_rotate_oracle),
    bootstrap_glwe_lut_extract=functools.partial(M.bootstrap_glwe_lut_extract, rotate=M.blind_rotate_oracle))
MB = dict(ref=EXACT, layout=F.paired)

THRESHOLDS = ('NUFHE_B200_WIDE_MAX', 'NUFHE_B200_WIDE2_MAX', 'NUFHE_B200_PAIR_MAX')
SCHEDULES = {'default': {}, 'stagger0': {'NUFHE_B200_STAGGER': '0'}, 'one_chunk': {'NUFHE_B200_MAX_CHUNKS': '1'},
             'force_odd': {'NUFHE_B200_FORCE_CHUNKS': '5'}, 'force4': {'NUFHE_B200_FORCE_CHUNKS': '4'},
             'thresholds': {k: '1000000' for k in THRESHOLDS}}
KNOBS = set(THRESHOLDS) | {k for s in SCHEDULES.values() for k in s} | {'NUFHE_B200_PAIR_ASYNC', 'NUFHE_B200_FFT'}


@functools.lru_cache(None)
def wave():
    return 4 * torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def engine(monkeypatch, schedule='default'):
    """an Engine whose context read the schedule's knobs (a context reads them when it is created)"""
    from nufhe_b200.engine import Engine
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in SCHEDULES[schedule].items():
        monkeypatch.setenv(k, v)
    return Engine()


def batches(schedule, pairs=False):
    """ciphertext batches around one wave, or (pairs) extract2 job batches whose 2 B ciphertexts sit around it; the
    stagger applies to single waves only, the chunk schedules to multi-wave launches"""
    W = wave()
    if pairs:
        half = W // 2
        sizes = sorted({1, 3, W + 1} | ({half} if half % 2 else {half - 1, half + 1}))
        count = [2 * b for b in sizes]
    else:
        sizes = [1, 2, 3, W - 1, W, W + 1, 2 * W + 3]
        count = sizes
    if schedule == 'stagger0':
        return [b for b, c in zip(sizes, count) if c <= W]
    if schedule in ('one_chunk', 'force_odd', 'force4'):
        return [b for b, c in zip(sizes, count) if c > W]
    return sizes


def max_batch(pairs=False):
    return wave() + 1 if pairs else 2 * wave() + 3


def run_modes(eng, bk, modes, sizes_of, what):
    for mode in modes:
        dev = mode.upload(eng)
        for b in sizes_of(mode):
            mode.check(mode.call(eng, dev, bk, b), b, what)


def mb_key(keys, seed):
    """a noisy multi-bit key of keys' secrets, as the transformed rows (3n/2, 2, 2, 2, N) the oracle and the engine
    take"""
    return M.multibit_key(keys, seed)[1]


# ---- n = 26: the full matrix ----------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def n26():
    keys = O.OracleKeys(SEED, n=26, make_bk=False)
    n, bk, B, J = 26, mb_key(keys, SEED + 1), max_batch(), max_batch(pairs=True)
    t = O.phase_to_t32
    modes = [gate_mode('nand', n, bk, t(1, 8), -1, -1, 2**29, True, 2001, B, **MB),
             gate_mode('xor_mu_min', n, bk, t(1, 4), 2, 2, -2**31, True, 2002, B, **MB),
             gate_mode('andny', n, bk, t(-1, 8), -1, 1, 2**29, True, 2003, B, **MB),
             gate_mode('one_input', n, bk, 777777, -1, 9, 123456789, False, 2004, B, **MB),
             x2_mode('mux_jobs', n, bk, (t(-1, 8), 1, 1, True), (t(1, 8) + 4321, -1, 3, True), 2**29, 2005, J, **MB),
             x2_mode('job_b_one_input', n, bk, (t(-1, 8), 1, 1, True), (-55555, 3, 7, False), 123456789, 2006, J, **MB)]
    for L in (0, 1, 2):
        for per_ct in (False, True):
            for two in (False, True):
                modes.append(lut_mode('lut_L%d_%s_%s' % (L, 'stride1024' if per_ct else 'stride0',
                                                         'in2' if two else 'no_in2'),
                                      n, bk, L, per_ct, two, 2100 + 4 * L + 2 * per_ct + two, B, **MB))
    modes.append(glwe_mode('glwe', n, bk, 2200, B, **MB))
    return bk, modes


CELLS = ['default', 'stagger0', 'one_chunk', 'force_odd', 'thresholds']


@pytest.mark.parametrize('schedule', CELLS)
def test_matrix_n26(monkeypatch, n26, schedule):
    """n = 26 (13 groups): every mode at every batch of the cell, every output row compared"""
    ref, modes = n26
    eng = engine(monkeypatch, schedule)
    bk = eng.bk_prepare_multibit(eng.to_device(ref))
    run_modes(eng, bk, modes, lambda mode: batches(schedule, pairs=mode.kind == 'x2'), 'n=26 ' + schedule)


# ---- n = 500: the shipped dimension ---------------------------------------------------------------------------------

N500_FULL = (1, 5, 301)


def sample_rows(B):
    """16 rows of a large batch: the first two, the last three and random ones"""
    rows = {0, 1, B - 3, B - 2, B - 1}
    rng = G.rs(B)
    while len(rows) < 16:
        rows.add(int(rng.randint(0, B)))
    return sorted(rows)


@pytest.fixture(scope='module')
def n500():
    """NAND on real encryptions (also key-switched and decrypted), extract2 with distinct jobs, LUT at L = 0 and 2 with
    per-ciphertext test vectors, GLWE; the oracle on rows 0 .. 300 and 16 rows of 2W + 3"""
    keys = O.OracleKeys(SEED + 2)
    n, bk, B = 500, mb_key(keys, SEED + 3), max_batch()
    rows = numpy.array(sorted(set(range(N500_FULL[-1])) | set(sample_rows(B))))
    rng = G.rs(2300)
    bits = rng.randint(0, 2, (2, B)).astype(bool)
    x1, x2 = keys.encrypt(bits[0]), keys.encrypt(bits[1])
    num, den, sa, sb = O.GATE_TABLE['nand']
    nand = gate_mode('nand', n, bk, O.phase_to_t32(num, den), sa, sb, int(O.MU), True, 0, B, rows, x=(x1, x2), ref=EXACT)
    nand.truth = ~(bits[0] & bits[1])
    t = O.phase_to_t32
    modes = [nand,
             x2_mode('mux_jobs', n, bk, (t(-1, 8), 1, 1, True), (t(1, 8) + 4321, -1, 3, True), 2**29, 2301, B, rows,
                     **MB),
             lut_mode('lut_L0', n, bk, 0, True, True, 2302, B, rows, **MB),
             lut_mode('lut_L2', n, bk, 2, True, True, 2303, B, rows, **MB),
             glwe_mode('glwe', n, bk, 2304, B, rows, **MB)]
    return keys, bk, modes


@pytest.mark.parametrize('schedule', ['default', 'force4'])
def test_matrix_n500(monkeypatch, n500, schedule):
    """n = 500 at B = 1, 5, 301 (every row compared) and 2W + 3 (16 rows compared); with 4 forced chunks (2W + 3 only)
    the chains resume at groups 63, 126 and 189.  The NAND outputs also decrypt to the truth table after the key
    switch."""
    keys, ref, modes = n500
    eng = engine(monkeypatch, schedule)
    bk = eng.bk_prepare_multibit(eng.to_device(ref))
    sizes = (list(N500_FULL) if schedule == 'default' else []) + [2 * wave() + 3]
    run_modes(eng, bk, modes, lambda mode: sizes, 'n=500 ' + schedule)
    nand = modes[0]
    dev = nand.upload(eng)
    ks = tuple(eng.to_device(x) for x in keys.ks)
    for b in sizes:
        ext = nand.call(eng, dev, bk, b)
        ra, rb, _ = eng.keyswitch(ks, (eng.to_device(ext[0]), eng.to_device(ext[1])))
        assert (keys.decrypt((eng.to_host(ra), eng.to_host(rb))) == nand.truth[:b]).all(), (schedule, b)


# ---- n = 2 (one group) and n = 1024 (LWE_N_MAX, 512 groups) ---------------------------------------------------------

@pytest.fixture(scope='module')
def dims():
    """n = 2: gate, LUT and GLWE up to 2W + 3 (the first 144 rows hold every pair of targets); n = 1024: gate, LUT
    (L = 2, per ciphertext) and GLWE at B = 3 on a random integral key"""
    keys = O.OracleKeys(SEED + 4, n=2, make_bk=False)
    small_bk, B = mb_key(keys, SEED + 5), max_batch()
    t = O.phase_to_t32
    small = [gate_mode('nand', 2, small_bk, t(1, 8), -1, -1, 2**29, True, 2401, B, **MB),
             lut_mode('lut_L1', 2, small_bk, 1, True, True, 2402, B, **MB),
             glwe_mode('glwe', 2, small_bk, 2403, B, **MB)]
    big_bk = O.bk_transform(G.torus32(G.rs(2404), (1536, 2, 2, 2, N)))
    big = [gate_mode('nand', 1024, big_bk, t(1, 8), -1, -1, 2**29, True, 2405, 3, **MB),
           lut_mode('lut_L2', 1024, big_bk, 2, True, True, 2406, 3, **MB),
           glwe_mode('glwe', 1024, big_bk, 2407, 3, **MB)]
    return (small_bk, small, [1, 2, 3, wave() + 1, 2 * wave() + 3]), (big_bk, big, [3])


def test_matrix_dimensions(monkeypatch, dims):
    eng = engine(monkeypatch)
    for ref, modes, sizes in dims:
        bk = eng.bk_prepare_multibit(eng.to_device(ref))
        run_modes(eng, bk, modes, lambda mode: sizes, 'n=%d' % modes[0].n)
        del bk


# ---- worst-case keys, digits and rotations --------------------------------------------------------------------------

ROT_PAIRS = [(N, 0), (N // 2, N // 2), (N, N), (1, N - 1), (2 * N - 1, N + 1), (N, 2 * N - 1)]


def worst_key(groups, shift):
    """raw rows at the extremes of the 32-bit range: -2^31, 2^31 - 1, alternating and -2^31 + 2^15, one pattern per
    polynomial, cycled from `shift`"""
    idx = numpy.arange(N)
    pats = [numpy.full(N, -2**31), numpy.full(N, 2**31 - 1), numpy.where(idx % 2, -2**31, 2**31 - 1),
            numpy.full(N, -2**31 + 2**15)]
    raw = numpy.empty((3 * groups, 2, 2, 2, N), numpy.int32)
    for i, ix in enumerate(numpy.ndindex(raw.shape[:-1])):
        raw[ix] = pats[(i + shift) % len(pats)]
    return O.bk_transform(raw)


def worst_inputs(n):
    """b = 0 (so the first group decomposes the test vector itself) and a = abar << 21 with the groups' rotation
    pairs cycling through ROT_PAIRS; GLWE test vectors whose digits are all -512, all 511, alternating, or -512 in the
    mask and 511 in the body"""
    lo = (-(2**31 + 2**21)) % 2**32                   # t = acc + 2^31 + 2^21 = 0: every digit -512
    hi = (0xfffff000 - (2**31 + 2**21)) % 2**32       # t = 0xfffff000: every digit 511
    alt = numpy.where(numpy.arange(N) % 2, lo, hi)
    tvs = [(lo, lo), (hi, hi), (alt, alt), (lo, hi)]
    B = len(tvs) * len(ROT_PAIRS)
    tv = numpy.empty((B, 2, N), numpy.int64)
    a = numpy.empty((B, n), numpy.int64)
    for r in range(B):
        tv[r, 0], tv[r, 1] = tvs[r // len(ROT_PAIRS)]
        for g in range(n // 2):
            a[r, 2 * g:2 * g + 2] = ROT_PAIRS[(r + g) % len(ROT_PAIRS)]
    return (F.i32(a << 21), numpy.zeros(B, numpy.int32)), F.i32(tv)


@pytest.mark.parametrize('n', [2, 8])
def test_worst_case_inputs(monkeypatch, n):
    """keys at the extremes of the 32-bit range, digits at -512 / 511 and rotations whose factors X^k - 1 reach -2, on
    the device against the exact oracle (the float reference has no margin here)"""
    eng = engine(monkeypatch)
    x, tv = worst_inputs(n)
    assert (O.t32_to_phase(x[0], 2 * N) == x[0].view(numpy.uint32) >> 21).all()
    for shift in range(4):
        ref = worst_key(n // 2, shift)
        bk = eng.bk_prepare_multibit(eng.to_device(ref))
        got = eng.bootstrap_glwe_lut_extract((eng.to_device(x[0]), eng.to_device(x[1])), eng.to_device(tv), bk)
        want = EXACT.bootstrap_glwe_lut_extract(x, tv, ref)
        assert numpy.array_equal(eng.to_host(got[0]), want[0]), (n, shift)
        assert numpy.array_equal(eng.to_host(got[1]).reshape(-1), want[1]), (n, shift)


# ---- the C ABI with a multi-bit key ---------------------------------------------------------------------------------

def test_c_abi_refusals(monkeypatch):
    """NB_EINVAL for an odd n, for a key with fewer than n / 2 groups and for a key that is not integral; NB_EUNSUPPORTED
    for the explicit-accumulator calls"""
    eng = engine(monkeypatch)
    lib, h = eng.lib, eng.handle
    keys = O.OracleKeys(SEED + 6, n=4, make_bk=False)
    bk = eng.bk_prepare_multibit(eng.to_device(mb_key(keys, SEED + 7)))           # 2 groups
    B = 2
    a = eng.to_device(G.torus32(G.rs(2500), (B, 6)))
    b = eng.to_device(G.torus32(G.rs(2501), (B,)))
    oa, ob = eng.empty((B, N), torch.int32), eng.empty((B,), torch.int32)

    def extract(n):
        rc = lib.nb_bootstrap_extract(h, ptr(a), ptr(b), None, None, 0, 1, 0, 2**29, ptr(bk), n, ptr(oa), ptr(ob), B)
        torch.cuda.synchronize()
        return rc
    assert extract(3) == _native.NB_EINVAL                     # odd n
    assert extract(6) == _native.NB_EINVAL                     # 3 groups wanted, 2 prepared
    assert extract(4) == _native.NB_OK
    acc = eng.to_device(numpy.zeros((B, 2, N), numpy.int32))
    bara = eng.to_device(numpy.zeros((B, 4), numpy.int32))
    oacc = eng.empty((B, 2, N), torch.int32)
    assert lib.nb_blind_rotate(h, ptr(acc), ptr(bara), ptr(bk), 4, ptr(oa), ptr(ob), ptr(oacc), B) == _native.NB_EUNSUPPORTED
    assert lib.nb_external_product(h, ptr(acc), ptr(bk), 0, B) == _native.NB_EUNSUPPORTED
    # field elements that are no transform of a centred 32-bit integer key
    bad = eng.to_device(G.rs(2502).randint(0, 2**62, size=(6, 2, 2, 2, N), dtype=numpy.int64))
    out = eng.empty((6, lib.nb_bk_multibit_row_u64()), torch.int64)
    assert lib.nb_bk_prepare_multibit(h, ptr(bad), ptr(out), 2) == _native.NB_EINVAL
    torch.cuda.synchronize()


def test_re_registration(monkeypatch):
    """a buffer prepared as a multi-bit key and then as a standard key is a standard key (the gate gives the standard
    oracle's bits), and the other way round a multi-bit key (the exact multi-bit oracle's bits)"""
    eng = engine(monkeypatch)
    keys = O.OracleKeys(SEED + 8, n=4, make_bk=False)
    std = M.standard_key(keys, SEED + 9)[1]
    mbk = mb_key(keys, SEED + 10)
    words = max(4 * eng.lib.nb_bk_row_u64(), 6 * eng.lib.nb_bk_multibit_row_u64())
    buf = eng.empty((words,), torch.int64)
    t = O.phase_to_t32
    B = 8
    want_std = gate_mode('nand', 4, std, t(1, 8), -1, -1, 2**29, True, 2600, B)
    want_mb = gate_mode('nand', 4, mbk, t(1, 8), -1, -1, 2**29, True, 2600, B, ref=EXACT)
    assert not want_std.equal(want_mb.want, B)
    dev = want_std.upload(eng)
    for first, second, mode in ((mbk, std, want_std), (std, mbk, want_mb)):
        for key in (first, second):
            name = 'nb_bk_prepare_multibit' if key is mbk else 'nb_bk_prepare'
            count = 2 if key is mbk else 4
            eng._call(name, ptr(eng.to_device(key)), ptr(buf), count)
        mode.check(mode.call(eng, dev, buf, B), B, 're-registration')
