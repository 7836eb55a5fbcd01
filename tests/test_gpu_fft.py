"""The FP64 step of the throughput shape on the GPU: forced on small and ragged batches, it gives the bits of the NTT
step and of the oracle; it really is the FP64 step that runs (it reads the key spectra); a key with random field
coefficients (no spectra) keeps the NTT step in the same shape."""
import numpy
import pytest

import gen_inputs as G
from oracle import oracle as O

pytestmark = pytest.mark.gpu


def _nand(eng, keys_bk, keys, a, b, spoil_spectra=False):
    bk_int = eng.bk_prepare(eng.to_device(keys_bk))
    if spoil_spectra:
        bk_int[:, eng.lib.nb_bk_row_u64() - 16 * 512 * 2:] = 0      # the FP64 part of every row (br_phases.cuh: BK_FFT_U64)
    ks = (eng.to_device(keys.ks_a), eng.to_device(keys.ks_b), eng.to_device(keys.ks_cv))
    num, den, sa, sb = O.GATE_TABLE['nand']
    ext = eng.bootstrap_extract((eng.to_device(a[0]), eng.to_device(a[1])), (eng.to_device(b[0]), eng.to_device(b[1])),
                                O.phase_to_t32(num, den), sa, sb, O.MU, bk_int)
    ra, rb, _ = eng.keyswitch(ks, ext)
    return eng.to_host(ra), eng.to_host(rb)


def test_fft_step_equals_ntt_step_and_oracle(monkeypatch):
    from nufhe_b200.engine import Engine
    keys = O.OracleKeys(G.GATE_SEED)
    rng = G.rs(481)
    monkeypatch.setenv('NUFHE_B200_WIDE_MAX', '0')      # the throughput shape at every batch
    monkeypatch.setenv('NUFHE_B200_WIDE2_MAX', '0')
    monkeypatch.setenv('NUFHE_B200_PAIR_MAX', '0')
    for B in (3, 700):
        bits_a, bits_b = rng.randint(0, 2, B).astype(bool), rng.randint(0, 2, B).astype(bool)
        a, b = keys.encrypt(bits_a), keys.encrypt(bits_b)
        outs = {}
        for fft in ('1', '0'):
            monkeypatch.setenv('NUFHE_B200_FFT', fft)
            outs[fft] = _nand(Engine(), keys.bk, keys, a, b)
        assert (outs['1'][0] == outs['0'][0]).all() and (outs['1'][1] == outs['0'][1]).all(), B
        assert (keys.decrypt(outs['1']) == ~(bits_a & bits_b)).all()
        sub = numpy.arange(0, B, max(1, B // 3))
        want = O.gate_binary('nand', (a[0][sub], a[1][sub]), (b[0][sub], b[1][sub]), keys.bk, keys.ks)
        assert (outs['1'][0][sub] == want[0]).all() and (outs['1'][1][sub] == want[1]).all()


def test_random_field_key_keeps_the_ntt_step(monkeypatch):
    """With a random field key the FP64 step would round garbage; the bits must be the NTT step's."""
    from nufhe_b200.engine import Engine
    keys = O.OracleKeys(G.GATE_SEED)
    rng = G.rs(482)
    bk = G.ff_numbers(rng, keys.bk.shape)
    monkeypatch.setenv('NUFHE_B200_WIDE_MAX', '0')
    monkeypatch.setenv('NUFHE_B200_WIDE2_MAX', '0')
    monkeypatch.setenv('NUFHE_B200_PAIR_MAX', '0')
    a, b = keys.encrypt(rng.randint(0, 2, 4).astype(bool)), keys.encrypt(rng.randint(0, 2, 4).astype(bool))
    outs = {}
    for fft in ('1', '0'):
        monkeypatch.setenv('NUFHE_B200_FFT', fft)
        outs[fft] = _nand(Engine(), bk, keys, a, b)
    assert (outs['1'][0] == outs['0'][0]).all() and (outs['1'][1] == outs['0'][1]).all()
    want = O.gate_binary('nand', a, b, bk, keys.ks)
    assert (outs['1'][0] == want[0]).all() and (outs['1'][1] == want[1]).all()


def test_throughput_shape_runs_the_fp64_step(monkeypatch):
    """With the key spectra zeroed after preparation the FP64 step must give wrong results and the NTT step (which
    does not read them) the oracle's: so the comparisons above are between two different kernels."""
    from nufhe_b200.engine import Engine
    keys = O.OracleKeys(G.GATE_SEED)
    rng = G.rs(483)
    monkeypatch.setenv('NUFHE_B200_WIDE_MAX', '0')
    monkeypatch.setenv('NUFHE_B200_WIDE2_MAX', '0')
    monkeypatch.setenv('NUFHE_B200_PAIR_MAX', '0')
    a, b = keys.encrypt(rng.randint(0, 2, 4).astype(bool)), keys.encrypt(rng.randint(0, 2, 4).astype(bool))
    want = O.gate_binary('nand', a, b, keys.bk, keys.ks)
    monkeypatch.setenv('NUFHE_B200_FFT', '0')
    got = _nand(Engine(), keys.bk, keys, a, b, spoil_spectra=True)
    assert (got[0] == want[0]).all() and (got[1] == want[1]).all()
    monkeypatch.setenv('NUFHE_B200_FFT', '1')
    got = _nand(Engine(), keys.bk, keys, a, b, spoil_spectra=True)
    assert not ((got[0] == want[0]).all() and (got[1] == want[1]).all())
