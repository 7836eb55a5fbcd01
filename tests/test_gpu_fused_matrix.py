"""Every entry point of the fused bootstrap in every CTA shape and schedule, bit for bit against the CPU oracle's
compositions (tests/fused_ref.py).

Shapes (forced through the shape thresholds, which a context reads when it is created, so one Engine per cell):
fp64 and ntt (2 ciphertexts per 256 threads, FP64 or NTT step), wide (1 ciphertext per 256 threads), wide2 (1 per 512
threads), pair and pair_barrier (1 per cluster of two CTAs, st.async or barrier exchange).  Schedules: the default;
no start-up stagger (single-wave launches of the 2-CTA-per-SM shapes); one chunk per chain and 4 forced chunks
(multi-wave launches of the queued shapes; at n = 25 the chunks start at steps 0, 7, 14 and 21, so two of them resume
on an odd step).  Batches are placed around one wave W of the shape.

Every call goes through the C ABI with its outputs inside larger buffers whose guard rows must keep their sentinel.
Edge rows come first in every input set: prologues whose mod-switch gives barb and bara in {0, 1, 1023, 1024, 1025,
2047}, the rounding ties of the LUT mod-switch (including the wrap near 2^32), and test-vector coefficients -2^31,
2^31 - 1 and 0 at indices 0 and 1023.  Every cell also repeats one call per mode on a key whose FP64 part is zeroed
(as in test_gpu_fft_kernels.py): where the FP64 step runs the result changes (an explicit rotation returns its input
accumulator, a plain product 0), where the NTT step runs it does not.  (A gate with mu = -2^31 is exempt: its
accumulator stays the constant -2^31 whatever the key.)

The oracle runs once per mode and dimension on the largest batch any cell uses; every cell compares its prefix."""
import functools

import numpy
import pytest
import torch

import gen_inputs as G
import fused_ref as F
from fused_ref import EDGE_ROT, Mode, gate_mode, glwe_mode, guarded, lut_mode, ptr, unguard, x2_mode
from oracle import oracle as O

pytestmark = pytest.mark.gpu
N = 1024
FFT_U64 = 16 * 512 * 2                      # the FP64 part at the end of every engine key row

# (WIDE_MAX, WIDE2_MAX, PAIR_MAX, PAIR_ASYNC, FFT)
SHAPES = {'fp64': ('0', '0', '0', '1', '1'), 'ntt': ('0', '0', '0', '1', '0'),
          'wide': ('1000000', '0', '0', '1', '1'), 'wide2': ('1000000', '1000000', '0', '1', '1'),
          'pair': ('0', '0', '1000000', '1', '1'), 'pair_barrier': ('0', '0', '1000000', '0', '1')}
SCHEDULES = {'default': {}, 'stagger0': {'NUFHE_B200_STAGGER': '0'}, 'one_chunk': {'NUFHE_B200_MAX_CHUNKS': '1'},
             'force4': {'NUFHE_B200_FORCE_CHUNKS': '4'}}
CELLS = ([(s, 'default') for s in SHAPES] + [(s, 'stagger0') for s in ('fp64', 'ntt', 'wide')]
         + [(s, sch) for s in ('fp64', 'ntt', 'wide', 'wide2') for sch in ('one_chunk', 'force4')])


@functools.lru_cache(None)
def sm_count():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def wave(shape):
    """ciphertexts in one wave of resident CTAs (pair: about one cluster per two SMs)"""
    return {'fp64': 4, 'ntt': 4, 'wide': 2, 'wide2': 1}.get(shape, 0.5) * sm_count() // 1


def batches(shape, schedule, pairs=False):
    """the batches of a cell: ciphertexts, or (pairs) the job batches of extract2, whose 2 B ciphertexts are placed
    around the wave; the stagger applies to single waves only, the chunk schedules to multi-wave launches"""
    W = int(wave(shape))
    if pairs:
        half = W // 2
        sizes = sorted({1, 3, W + 1} | ({half} if half % 2 else {half - 1, half + 1}))
        count = [2 * b for b in sizes]
    else:
        sizes = [1, 2, 3, W - 1, W, W + 1, 2 * W + 3]
        count = sizes
    if schedule == 'stagger0':
        return [b for b, c in zip(sizes, count) if c <= W]
    if schedule in ('one_chunk', 'force4'):
        return [b for b, c in zip(sizes, count) if c > W]
    return sizes


def max_batch(pairs=False):
    return 4 * sm_count() + 1 if pairs else 8 * sm_count() + 3


def engine(monkeypatch, shape, schedule='default'):
    from nufhe_b200.engine import Engine
    names = ('NUFHE_B200_WIDE_MAX', 'NUFHE_B200_WIDE2_MAX', 'NUFHE_B200_PAIR_MAX', 'NUFHE_B200_PAIR_ASYNC',
             'NUFHE_B200_FFT')
    for k in list(names) + [k for s in SCHEDULES.values() for k in s]:
        monkeypatch.delenv(k, raising=False)
    for k, v in zip(names, SHAPES[shape]):
        monkeypatch.setenv(k, v)
    for k, v in SCHEDULES[schedule].items():
        monkeypatch.setenv(k, v)
    return Engine()


def prepare(eng, bk):
    """the prepared key and a second preparation whose FP64 part is zeroed in place (it stays registered)"""
    bk_int = eng.bk_prepare(eng.to_device(bk))
    spoiled = eng.bk_prepare(eng.to_device(bk))
    spoiled[:, -FFT_U64:] = 0
    return bk_int, spoiled


def runs_fp64(shape, kind):
    """whether a call of this kind takes the FP64 step in this shape (integral keys only): the throughput shape with
    FFT = 1, which is also where a plain product goes in the pair shapes (they have no plain variant)"""
    return shape == 'fp64' or (shape.startswith('pair') and kind == 'plain')


# ---- modes only the standard key has ----------------------------------------------------------------------------

def explicit_mode(name, n, bk, seed, B):
    rng = G.rs(seed)
    acc = G.torus32(rng, (B, 2, N))
    bara = G.torus32(rng, (B, n), 0, 2 * N)
    m = min(bara.size, 8 * n)
    bara.reshape(-1)[:m] = numpy.resize(EDGE_ROT, m)
    wa, wb, wacc = F.blind_rotate(acc, bara, bk)

    def call(eng, dev, bk_int, b):
        dacc, dbara = dev
        oa, ob, oacc = guarded(eng, b, N), guarded(eng, b, 1), guarded(eng, b, 2 * N)
        eng._call('nb_blind_rotate', dacc.data_ptr(), dbara.data_ptr(), bk_int.data_ptr(), n, oa[F.GUARD].data_ptr(),
                  ob[F.GUARD].data_ptr(), oacc[F.GUARD].data_ptr(), b)
        return unguard(oa, 'out_a'), unguard(ob, 'out_b')[:, 0], unguard(oacc, 'accum_out').reshape(b, 2, N)
    mode = Mode(name, 'explicit', n, (wa, wb, wacc), numpy.arange(B),
                lambda eng: (eng.to_device(acc), eng.to_device(bara)), call)
    mode.acc = acc
    return mode


def plain_mode(name, n, bk, seed, B):
    rng = G.rs(seed)
    acc = G.torus32(rng, (B, 2, N))
    row = n - 1
    want = F.external_product(acc, bk, row)

    def call(eng, dev, bk_int, b):
        buf = guarded(eng, b, 2 * N)
        buf[F.GUARD:F.GUARD + b] = dev[:b].reshape(b, 2 * N)
        eng._call('nb_external_product', buf[F.GUARD].data_ptr(), bk_int.data_ptr(), row, b)
        return (unguard(buf, 'accum').reshape(b, 2, N),)
    return Mode(name, 'plain', n, (want,), numpy.arange(B), lambda eng: eng.to_device(acc), call)


# ---- running a cell -------------------------------------------------------------------------------------------------

def run_modes(eng, bk_int, spoiled, shape, modes, sizes_of, what):
    """every mode at every batch of the cell, then its largest batch again on the spoiled key"""
    for mode in modes:
        dev = mode.upload(eng)
        sizes = sizes_of(mode)
        for b in sizes:
            mode.check(mode.call(eng, dev, bk_int, b), b, what)
        b = sizes[-1]
        got = mode.call(eng, dev, spoiled, b)
        if not runs_fp64(shape, mode.kind) or mode.key_free:
            mode.check(got, b, what + ' (spoiled key, NTT step)')
        else:
            assert not mode.equal(got, b), (what, mode.name, b, 'the spoiled key gave the right bits: no FP64 step')
            if mode.kind == 'explicit':
                assert (got[2] == mode.acc[:b]).all(), (what, mode.name, b)
            if mode.kind == 'plain':
                assert (got[0] == 0).all(), (what, mode.name, b)


@pytest.fixture(scope='module')
def keys():
    return O.OracleKeys(G.GATE_SEED)


@pytest.fixture(scope='module')
def n25(keys):
    """the full matrix's modes at n = 25, each on the largest batch any cell uses"""
    n, bk, B, J = 25, keys.bk, max_batch(), max_batch(pairs=True)
    t = O.phase_to_t32
    modes = [gate_mode('nand', n, bk, t(1, 8), -1, -1, 2**29, True, 1001, B),
             gate_mode('xor', n, bk, t(1, 4), 2, 2, -2**31, True, 1002, B),
             gate_mode('xnor', n, bk, t(-1, 4), -2, -2, 2**29, True, 1003, B),
             gate_mode('andny', n, bk, t(-1, 8), -1, 1, 2**29, True, 1004, B),
             gate_mode('one_input', n, bk, 777777, -1, 9, 123456789, False, 1005, B),
             x2_mode('mux_jobs', n, bk, (t(-1, 8), 1, 1, True), (t(1, 8) + 4321, -1, 3, True), 2**29, 1006, J),
             x2_mode('job_b_one_input', n, bk, (t(-1, 8), 1, 1, True), (-55555, 3, 7, False), 123456789, 1007, J)]
    for L in (0, 1, 2):
        for per_ct in (False, True):
            for two in (False, True):
                modes.append(lut_mode('lut_L%d_%s_%s' % (L, 'stride1024' if per_ct else 'stride0',
                                                         'in2' if two else 'no_in2'),
                                      n, bk, L, per_ct, two, 1100 + 4 * L + 2 * per_ct + two, B))
    modes += [glwe_mode('glwe', n, bk, 1200, B), explicit_mode('explicit', n, bk, 1201, B),
              plain_mode('plain', n, bk, 1202, B)]
    return modes


@pytest.mark.parametrize('shape,schedule', CELLS, ids=['%s-%s' % c for c in CELLS])
def test_matrix_n25(monkeypatch, keys, n25, shape, schedule):
    """n = 25 (the gate key's first rows): every mode at every batch of the cell, every output row compared"""
    eng = engine(monkeypatch, shape, schedule)
    bk_int, spoiled = prepare(eng, keys.bk[:25])
    run_modes(eng, bk_int, spoiled, shape, n25, lambda mode: batches(shape, schedule, pairs=mode.kind == 'x2'),
              '%s/%s n=25' % (shape, schedule))


# ---- n = 500: the shipped dimension ---------------------------------------------------------------------------------

N500_FULL = (1, 5, 301)


def sample_rows(B):
    """16 rows of a large batch: the first two, the last, the two before it (the last full 2-ciphertext CTA) and
    random ones"""
    rows = {0, 1, B - 3, B - 2, B - 1}
    rng = G.rs(B)
    while len(rows) < 16:
        rows.add(int(rng.randint(0, B)))
    return sorted(rows)


def n500_rows():
    big = sorted({2 * int(wave(s)) + 3 for s in SHAPES})
    return numpy.array(sorted(set(range(N500_FULL[-1])).union(*[sample_rows(B) for B in big])))


@pytest.fixture(scope='module')
def n500(keys):
    """gate (NAND on real encryptions, also key-switched and decrypted), extract2 with distinct jobs, LUT at L = 0
    and 2 with per-ciphertext test vectors, GLWE; the oracle on the rows n500_rows() of the largest batch"""
    n, bk, B = 500, keys.bk, max_batch()
    rows = n500_rows()
    rng = G.rs(1300)
    bits = rng.randint(0, 2, (2, B)).astype(bool)
    x1, x2 = keys.encrypt(bits[0]), keys.encrypt(bits[1])
    num, den, sa, sb = O.GATE_TABLE['nand']
    nand = gate_mode('nand', n, bk, O.phase_to_t32(num, den), sa, sb, int(O.MU), True, 0, B, rows, x=(x1, x2))
    nand.truth = ~(bits[0] & bits[1])
    t = O.phase_to_t32
    return [nand,
            x2_mode('mux_jobs', n, bk, (t(-1, 8), 1, 1, True), (t(1, 8) + 4321, -1, 3, True), 2**29, 1301, B, rows),
            lut_mode('lut_L0', n, bk, 0, True, True, 1302, B, rows),
            lut_mode('lut_L2', n, bk, 2, True, True, 1303, B, rows),
            glwe_mode('glwe', n, bk, 1304, B, rows)]


@pytest.mark.parametrize('shape', list(SHAPES))
def test_matrix_n500(monkeypatch, keys, n500, shape):
    """n = 500 at B = 1, 5, 301 (every row compared) and 2W + 3 (16 rows compared); the NAND outputs also decrypt to
    the truth table after the key switch at every batch"""
    eng = engine(monkeypatch, shape)
    bk_int, spoiled = prepare(eng, keys.bk)
    ks = tuple(eng.to_device(x) for x in keys.ks)
    sizes = list(N500_FULL) + [2 * int(wave(shape)) + 3]
    run_modes(eng, bk_int, spoiled, shape, n500, lambda mode: sizes, '%s n=500' % shape)
    nand = n500[0]
    dev = nand.upload(eng)
    for b in sizes:
        ext = nand.call(eng, dev, bk_int, b)
        ra, rb, _ = eng.keyswitch(ks, (eng.to_device(ext[0]), eng.to_device(ext[1])))
        assert (keys.decrypt((eng.to_host(ra), eng.to_host(rb))) == nand.truth[:b]).all(), (shape, b)


# ---- n = 1024 (LWE_N_MAX) and n = 1 ---------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def dims(keys):
    """B = 3: gate, LUT (L = 2, per ciphertext) and GLWE at n = 1024 on a random integral key (so the FP64 step
    applies); gate and explicit rotation at n = 1 on the gate key's first row"""
    rng = G.rs(1400)
    bk = O.bk_transform(G.torus32(rng, (1024, 2, 2, 2, N)))
    t = O.phase_to_t32
    big = [gate_mode('nand', 1024, bk, t(1, 8), -1, -1, 2**29, True, 1401, 3),
           lut_mode('lut_L2', 1024, bk, 2, True, True, 1402, 3),
           glwe_mode('glwe', 1024, bk, 1403, 3)]
    small = [gate_mode('xor', 1, keys.bk, t(1, 4), 2, 2, -2**31, True, 1404, 3),
             explicit_mode('explicit', 1, keys.bk, 1405, 3)]
    return bk, big, small


@pytest.mark.parametrize('shape', list(SHAPES))
def test_matrix_dimensions(monkeypatch, keys, dims, shape):
    bk, big, small = dims
    eng = engine(monkeypatch, shape)
    for key, modes, n in ((bk, big, 1024), (keys.bk[:1], small, 1)):
        bk_int, spoiled = prepare(eng, key)
        run_modes(eng, bk_int, spoiled, shape, modes, lambda mode: [3], '%s n=%d' % (shape, n))
        del bk_int, spoiled
