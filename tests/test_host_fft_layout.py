"""Shared-memory layout of the FP64 CMux step (csrc/fft_layout.cuh), through the index functions the kernel itself uses
(compiled into the host emulator): every pass touches every spectrum position exactly once, and every 16-byte
warp-instruction of every pass is free of bank conflicts -- 4 wavefronts for the 512 bytes of a warp.  Also: the key
loads of pass 3 read contiguous 16-byte values, one per pair of ciphertext lanes."""
import ctypes
import os

import numpy
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
THREADS = 256                   # BrFft: 2 ciphertexts on 256 threads
SPECTRA = 8                     # 4 per ciphertext
PASSES = {0: 'fwd1 / inv1', 1: 'fwd2 / inv2', 2: 'pass 3 (DFT4, MAC, inverse DFT4)'}


@pytest.fixture(scope='module')
def emul():
    path = os.path.join(ROOT, 'nufhe_b200', 'csrc', 'libnb_host_emul.so')
    if not os.path.exists(path):
        import __graft_entry__ as g
        g.build()
    return ctypes.CDLL(path)


def _offsets(emul, phase):
    """(THREADS, instructions) array of the 16-byte offsets each thread touches, in program order"""
    buf = numpy.zeros(64, numpy.int32)
    rows = []
    for tid in range(THREADS):
        n = emul.emul_fft_smem_offsets(ctypes.c_int(phase), ctypes.c_int(tid), buf.ctypes.data_as(ctypes.c_void_p))
        rows.append(buf[:n].copy())
    return numpy.array(rows)


def _wavefronts(lane_offsets):
    """128-bit shared-memory accesses are served one quarter warp (8 lanes, 128 bytes) at a time; inside a quarter,
    distinct 16-byte addresses in the same bank group (offset mod 8) are serialised, equal ones are broadcast"""
    total = 0
    for q in range(4):
        quarter = lane_offsets[8 * q:8 * q + 8]
        per_group = {}
        for off in set(int(x) for x in quarter):
            per_group[off % 8] = per_group.get(off % 8, 0) + 1
        total += max(per_group.values())
    return total


@pytest.mark.parametrize('phase', sorted(PASSES))
def test_every_pass_touches_every_position_once(emul, phase):
    flat = _offsets(emul, phase).reshape(-1)
    assert flat.size == SPECTRA * 512 and numpy.unique(flat).size == flat.size, PASSES[phase]


@pytest.mark.parametrize('phase', sorted(PASSES))
def test_every_warp_instruction_takes_four_wavefronts(emul, phase):
    off = _offsets(emul, phase)
    for w in range(THREADS // 32):
        for i in range(off.shape[1]):
            assert _wavefronts(off[32 * w:32 * w + 32, i]) == 4, (PASSES[phase], w, i)


def test_positions_fit_the_padded_spectra(emul):
    """all passes address the same 8 x 512 positions, inside the 8 padded spectra the kernel allocates
    (fft_layout.cuh: FFT_SPEC_CPLX = 522 complex values each)"""
    sets = [set(_offsets(emul, p).reshape(-1).tolist()) for p in PASSES]
    assert sets[0] == sets[1] == sets[2]
    assert min(sets[0]) >= 0 and max(sets[0]) < SPECTRA * 522


def test_key_loads_of_a_warp_are_contiguous(emul):
    """pass 3: lanes 2 i and 2 i + 1 (the two ciphertexts of one group) read the same key value, and the 16 groups of a
    warp read 16 consecutive values -- 256 contiguous bytes per warp-instruction"""
    for w in range(THREADS // 32):
        for ks in range(16):
            for k3 in range(4):
                o = numpy.array([emul.emul_fft_key_offset(32 * w + l, ks, k3) for l in range(32)])
                assert (o[0::2] == o[1::2]).all()
                assert (numpy.diff(o[0::2]) == 1).all(), (w, ks, k3)
                assert o[0] % 16 == 0
    seen = {emul.emul_fft_key_offset(t, ks, k3) for t in range(0, THREADS, 2) for ks in range(16) for k3 in range(4)}
    assert seen == set(range(16 * 512))
