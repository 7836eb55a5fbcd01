"""Gate-level parity on the GPU: fused bootstrap + key switch through the C ABI against
(1) the committed output of the reference's own closures (tests/golden/gate.npz) and
(2) the CPU oracle on larger batches, plus decryption truth tables (test/test_gates.py:40-85)."""
import numpy
import pytest
import torch

import gen_inputs as G
from oracle import oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def eng():
    from nufhe_b200.engine import Engine
    return Engine()


@pytest.fixture(scope='module')
def keys():
    return O.OracleKeys(G.GATE_SEED)


@pytest.fixture(scope='module')
def dev_keys(eng, keys):
    bk_int = eng.bk_prepare(eng.to_device(keys.bk))
    ks = (eng.to_device(keys.ks_a), eng.to_device(keys.ks_b), eng.to_device(keys.ks_cv))
    return bk_int, ks


def gpu_gate(eng, dev_keys, name, a, b):
    bk_int, ks = dev_keys
    num, den, sa, sb = O.GATE_TABLE[name]
    da = (eng.to_device(a[0]), eng.to_device(a[1]))
    db = (eng.to_device(b[0]), eng.to_device(b[1]))
    ext = eng.bootstrap_extract(da, db, O.phase_to_t32(num, den), sa, sb, O.MU, bk_int)
    ra, rb, _ = eng.keyswitch(ks, ext)
    return (eng.to_host(ext[0]), eng.to_host(ext[1])), (eng.to_host(ra), eng.to_host(rb))


def test_nand_matches_reference_closures(eng, keys, dev_keys, golden):
    g = golden('gate')
    c1 = (g['c1_a'][:2], g['c1_b'][:2])
    c2 = (g['c2_a'][:2], g['c2_b'][:2])
    ext, out = gpu_gate(eng, dev_keys, 'nand', c1, c2)
    assert (ext[0] == g['nand_ext_a']).all() and (ext[1] == g['nand_ext_b']).all()
    assert (out[0] == g['nand_a']).all() and (out[1] == g['nand_b']).all()
    assert (keys.decrypt(out) == g['nand_bits']).all()


@pytest.mark.parametrize('name,batch', [('nand', 1), ('nand', 37), ('xor', 8), ('andny', 5)])
def test_binary_gates_vs_oracle(eng, keys, dev_keys, name, batch):
    rng = G.rs(400 + batch)
    bits_a, bits_b = rng.randint(0, 2, batch).astype(bool), rng.randint(0, 2, batch).astype(bool)
    a, b = keys.encrypt(bits_a), keys.encrypt(bits_b)
    ext, out = gpu_gate(eng, dev_keys, name, a, b)
    want = O.gate_binary(name, a, b, keys.bk, keys.ks)
    assert (out[0] == want[0]).all() and (out[1] == want[1]).all()
    truth = dict(nand=~(bits_a & bits_b), xor=bits_a ^ bits_b, andny=~bits_a & bits_b)[name]
    assert (keys.decrypt(out) == truth).all()


def test_mux_vs_oracle(eng, keys, dev_keys):
    bk_int, ks = dev_keys
    rng = G.rs(450)
    B = 6
    bits = [rng.randint(0, 2, B).astype(bool) for _ in range(3)]
    a, b, c = (keys.encrypt(x) for x in bits)
    d = [(eng.to_device(x[0]), eng.to_device(x[1])) for x in (a, b, c)]
    and_const = O.phase_to_t32(-1, 8)
    u1 = eng.bootstrap_extract(d[0], d[1], and_const, 1, 1, O.MU, bk_int)
    u2 = eng.bootstrap_extract(d[0], d[2], and_const, -1, 1, O.MU, bk_int)
    ra, rb, _ = eng.keyswitch(ks, u1, u2, c=O.phase_to_t32(1, 8))
    want = O.gate_mux(a, b, c, keys.bk, keys.ks)
    assert (eng.to_host(ra) == want[0]).all() and (eng.to_host(rb) == want[1]).all()
    assert (keys.decrypt((eng.to_host(ra), eng.to_host(rb))) == numpy.where(bits[0], bits[1], bits[2])).all()


def test_nand_more_than_one_wave_vs_oracle(eng, keys, dev_keys):
    """600 ciphertexts = 300 CTAs > the 264 co-resident ones of an H100: exercises CTA turnover; every (a, b) is compared."""
    rng = G.rs(470)
    B = 600
    bits_a, bits_b = rng.randint(0, 2, B).astype(bool), rng.randint(0, 2, B).astype(bool)
    a, b = keys.encrypt(bits_a), keys.encrypt(bits_b)
    ext, out = gpu_gate(eng, dev_keys, 'nand', a, b)
    want = O.gate_binary('nand', a, b, keys.bk, keys.ks)
    assert (out[0] == want[0]).all() and (out[1] == want[1]).all()
    assert (keys.decrypt(out) == ~(bits_a & bits_b)).all()


@pytest.mark.parametrize('batch', [4096, 16384])
def test_full_size_batches_decrypt_to_truth_table(eng, keys, dev_keys, batch):
    """BASELINE.json batch sizes: size-independent property (encrypt -> gate -> decrypt == truth table) for
    NAND and MUX, plus determinism (two runs give identical ciphertexts) and batch-independence (the first
    37 outputs equal those of a 37-ciphertext run)."""
    bk_int, ks = dev_keys
    rng = G.rs(480 + batch)
    bits = [rng.randint(0, 2, batch).astype(bool) for _ in range(3)]
    cts = [keys.encrypt(x) for x in bits]
    d = [(eng.to_device(x[0]), eng.to_device(x[1])) for x in cts]
    num, den, sa, sb = O.GATE_TABLE['nand']
    ext = eng.bootstrap_extract(d[0], d[1], O.phase_to_t32(num, den), sa, sb, O.MU, bk_int)
    ra, rb, _ = eng.keyswitch(ks, ext)
    out = (eng.to_host(ra), eng.to_host(rb))
    assert (keys.decrypt(out) == ~(bits[0] & bits[1])).all()
    ext2 = eng.bootstrap_extract(d[0], d[1], O.phase_to_t32(num, den), sa, sb, O.MU, bk_int)
    ra2, rb2, _ = eng.keyswitch(ks, ext2)
    assert torch.equal(ra, ra2) and torch.equal(rb, rb2)
    small = [(x[0][:37].contiguous(), x[1][:37].contiguous()) for x in d[:2]]
    ext3 = eng.bootstrap_extract(small[0], small[1], O.phase_to_t32(num, den), sa, sb, O.MU, bk_int)
    ra3, rb3, _ = eng.keyswitch(ks, ext3)
    assert torch.equal(ra[:37], ra3) and torch.equal(rb[:37], rb3)
    and_const = O.phase_to_t32(-1, 8)
    u1, u2 = eng.bootstrap_extract2((d[0], d[1], and_const, 1, 1), (d[0], d[2], and_const, -1, 1), O.MU, bk_int)
    ma, mb, _ = eng.keyswitch(ks, u1, u2, c=O.phase_to_t32(1, 8))
    assert (keys.decrypt((eng.to_host(ma), eng.to_host(mb))) == numpy.where(bits[0], bits[1], bits[2])).all()


# ---- BASELINE.md section 4 parity set --------------------------------------------------------------------------

def test_nand32_and_mux_match_reference_closures(eng, keys, dev_keys, golden):
    """32 NAND ciphertexts and 4 MUX triples against tests/golden/gates32.npz -- inputs, extracted samples and final
    ciphertexts produced by the UNMODIFIED reference's NumPy closures (make_golden_gates32.py), same keys as
    gate.npz.  Bit-exact on every (a, b)."""
    g = golden('gates32')
    bk_int, ks = dev_keys
    ext, out = gpu_gate(eng, dev_keys, 'nand', (g['in1_a'], g['in1_b']), (g['in2_a'], g['in2_b']))
    assert (ext[0] == g['nand_ext_a']).all() and (ext[1] == g['nand_ext_b']).all()
    assert (out[0] == g['nand_a']).all() and (out[1] == g['nand_b']).all()
    assert (keys.decrypt(out) == ~(g['bits_a'] & g['bits_b'])).all()
    d = [(eng.to_device(g['mux_in_a'][i]), eng.to_device(g['mux_in_b'][i])) for i in range(3)]
    and_const = O.phase_to_t32(-1, 8)
    u1, u2 = eng.bootstrap_extract2((d[0], d[1], and_const, 1, 1), (d[0], d[2], and_const, -1, 1), O.MU, bk_int)
    assert (eng.to_host(u1[0]) == g['mux_u1_a']).all() and (eng.to_host(u1[1]) == g['mux_u1_b']).all()
    assert (eng.to_host(u2[0]) == g['mux_u2_a']).all() and (eng.to_host(u2[1]) == g['mux_u2_b']).all()
    ma, mb, _ = eng.keyswitch(ks, u1, u2, c=O.phase_to_t32(1, 8))
    assert (eng.to_host(ma) == g['mux_a']).all() and (eng.to_host(mb) == g['mux_b']).all()
    mb_ = g['mux_bits']
    assert (keys.decrypt((eng.to_host(ma), eng.to_host(mb))) == numpy.where(mb_[0], mb_[1], mb_[2])).all()


def test_vm_gate_mux_matches_reference_closures(golden):
    """The same MUX through the public API (Context -> VirtualMachine.gate_mux, nufhe/gates.py:600-664)."""
    import nufhe_b200 as nufhe
    from nufhe_b200.lwe import LweSampleArray
    g = golden('gates32')
    ctx = nufhe.Context(rng=nufhe.DeterministicRNG(G.GATE_SEED))
    sk, ck = ctx.make_key_pair()
    vm = ctx.make_virtual_machine(ck)
    thr = ctx.thread
    cts = [LweSampleArray(ck.params.in_out_params, thr.to_device(g['mux_in_a'][i]), thr.to_device(g['mux_in_b'][i]),
                          torch.zeros(4, dtype=torch.float32, device=thr.device)) for i in range(3)]
    r = vm.gate_mux(*cts)
    assert (r.a.cpu().numpy() == g['mux_a']).all() and (r.b.cpu().numpy() == g['mux_b']).all()


def test_full_4096_nand_and_mux_equal_the_oracle(eng, keys, dev_keys):
    """BASELINE.md section 4: bit-exact against the CPU oracle on ALL 4096 outputs, NAND and MUX (the oracle runs
    ~70 s + ~140 s on 16 host cores).  4096 x 500 steps x 8192 multiplications put a few elements on the rare path
    of the deferred canonicalisation (probability 2^-32 each), so this is also its end-to-end check."""
    bk_int, ks = dev_keys
    B = 4096
    rng = G.rs(4096)
    bits = [rng.randint(0, 2, B).astype(bool) for _ in range(3)]
    a, b, c = (keys.encrypt(x) for x in bits)
    ext, out = gpu_gate(eng, dev_keys, 'nand', a, b)
    want = O.gate_binary('nand', a, b, keys.bk, keys.ks)
    assert (out[0] == want[0]).all() and (out[1] == want[1]).all()
    d = [(eng.to_device(x[0]), eng.to_device(x[1])) for x in (a, b, c)]
    and_const = O.phase_to_t32(-1, 8)
    u1, u2 = eng.bootstrap_extract2((d[0], d[1], and_const, 1, 1), (d[0], d[2], and_const, -1, 1), O.MU, bk_int)
    ma, mb, _ = eng.keyswitch(ks, u1, u2, c=O.phase_to_t32(1, 8))
    want = O.gate_mux(a, b, c, keys.bk, keys.ks)
    assert (eng.to_host(ma) == want[0]).all() and (eng.to_host(mb) == want[1]).all()
    assert (keys.decrypt(want) == numpy.where(bits[0], bits[1], bits[2])).all()


def test_batch_65536_truth_table_and_strided_oracle_subset(eng, keys, dev_keys):
    """BASELINE.json config 5's batch on one GPU: every output decrypts to NAND, and a strided 512-ciphertext subset
    equals the oracle bit for bit."""
    B = 65536
    rng = G.rs(65536)
    bits_a, bits_b = rng.randint(0, 2, B).astype(bool), rng.randint(0, 2, B).astype(bool)
    a, b = keys.encrypt(bits_a), keys.encrypt(bits_b)
    ext, out = gpu_gate(eng, dev_keys, 'nand', a, b)
    assert (keys.decrypt(out) == ~(bits_a & bits_b)).all()
    sub = slice(17, None, 128)
    want = O.gate_binary('nand', (a[0][sub], a[1][sub]), (b[0][sub], b[1][sub]), keys.bk, keys.ks)
    assert (out[0][sub] == want[0]).all() and (out[1][sub] == want[1]).all()


@pytest.mark.parametrize('batch', [700, 1030])
def test_time_sliced_launches_equal_the_oracle(eng, keys, dev_keys, batch):
    """Batches between one and two waves are cut into chunks of steps that migrate between CTAs (accumulators parked
    in global memory, kernels.cuh: blind_rotate_kernel); every ciphertext must still equal the oracle."""
    rng = G.rs(batch)
    bits_a, bits_b = rng.randint(0, 2, batch).astype(bool), rng.randint(0, 2, batch).astype(bool)
    a, b = keys.encrypt(bits_a), keys.encrypt(bits_b)
    ext, out = gpu_gate(eng, dev_keys, 'nand', a, b)
    want = O.gate_binary('nand', a, b, keys.bk, keys.ks)
    assert (out[0] == want[0]).all() and (out[1] == want[1]).all()


def test_time_sliced_mux_equals_the_oracle(eng, keys, dev_keys):
    """gate_mux's double launch (two jobs in one kernel, nb_bootstrap_extract2) through the time-sliced queue: 2 x 330
    ciphertexts = 330 chains on 264 CTAs; and one batch in the time-sliced WIDE shape (2 x 200 ciphertexts)."""
    bk_int, ks = dev_keys
    and_const = O.phase_to_t32(-1, 8)
    for B in (330, 200):
        rng = G.rs(3300 + B)
        bits = [rng.randint(0, 2, B).astype(bool) for _ in range(3)]
        a, b, c = (keys.encrypt(x) for x in bits)
        d = [(eng.to_device(x[0]), eng.to_device(x[1])) for x in (a, b, c)]
        u1, u2 = eng.bootstrap_extract2((d[0], d[1], and_const, 1, 1), (d[0], d[2], and_const, -1, 1), O.MU, bk_int)
        ma, mb, _ = eng.keyswitch(ks, u1, u2, c=O.phase_to_t32(1, 8))
        want = O.gate_mux(a, b, c, keys.bk, keys.ks)
        assert (eng.to_host(ma) == want[0]).all() and (eng.to_host(mb) == want[1]).all(), B


_RARE_PATH_SCRIPT = r'''
import sys, numpy
sys.path.insert(0, %(root)r); sys.path.insert(0, %(root)r + '/tests/golden')
import gen_inputs as G
from oracle import oracle as O
from nufhe_b200.engine import Engine
eng = Engine()
keys = O.OracleKeys(G.GATE_SEED)
bk_int = eng.bk_prepare(eng.to_device(keys.bk))
ks = (eng.to_device(keys.ks_a), eng.to_device(keys.ks_b), eng.to_device(keys.ks_cv))
rng = G.rs(77)
B = 9
a, b = keys.encrypt(rng.randint(0, 2, B).astype(bool)), keys.encrypt(rng.randint(0, 2, B).astype(bool))
ext = eng.bootstrap_extract((eng.to_device(a[0]), eng.to_device(a[1])), (eng.to_device(b[0]), eng.to_device(b[1])),
                            O.phase_to_t32(1, 8), -1, -1, O.MU, bk_int)
ra, rb, _ = eng.keyswitch(ks, ext)
want = O.gate_binary('nand', a, b, keys.bk, keys.ks)
assert (eng.to_host(ra) == want[0]).all() and (eng.to_host(rb) == want[1]).all()
x = numpy.random.RandomState(5).randint(-2**31, 2**31, (64, 1024)).astype(numpy.int32)
f = eng.ntt_forward_i32(eng.to_device(x))
assert (eng.to_host(eng.ntt_inverse_i32(f)) == x).all()
# the LUT instantiations and the second job of extract2, against the oracle at n = 25
sys.path.insert(0, %(root)r + '/tests')
import fused_ref as F
bk25 = eng.bk_prepare(eng.to_device(keys.bk[:25]))
dev = lambda x: (eng.to_device(x[0]), eng.to_device(x[1]))
same = lambda got, want: all((eng.to_host(g) == w).all() for g, w in zip(got, want))
x1, x2, x3 = [(G.torus32(rng, (B, 25)), G.torus32(rng, (B,))) for _ in range(3)]
tv = G.torus32(rng, (B, 1024))
assert same(eng.bootstrap_lut_extract(dev(x1), dev(x2), 12345678, 2, -3, eng.to_device(tv), 2, bk25),
            F.bootstrap_lut_extract(x1, x2, 12345678, 2, -3, tv, 2, keys.bk))
tv2 = G.torus32(rng, (B, 2, 1024))
assert same(eng.bootstrap_glwe_lut_extract(dev(x1), eng.to_device(tv2), bk25), F.bootstrap_glwe_lut_extract(x1, tv2, keys.bk))
ja, jb = (x1, x2, O.phase_to_t32(-1, 8), 1, 1), (x3, x1, O.phase_to_t32(1, 8) + 4321, -1, 3)
u1, u2 = eng.bootstrap_extract2((dev(x1), dev(x2)) + ja[2:], (dev(x3), dev(x1)) + jb[2:], O.MU, bk25)
assert same(u1 + u2, F.bootstrap_extract(*ja, O.MU, keys.bk) + F.bootstrap_extract(*jb, O.MU, keys.bk))
print('rare path ok')
'''


@pytest.mark.parametrize('wide_max', ['throughput_fp64', 'throughput_ntt', '1000000', 'wide2', 'pair'])
def test_canonicalisation_rare_path_forced(wide_max):
    """NUFHE_B200_FORCE_RARE_PATH=1 lowers the trigger of the deferred canonicalisation so that EVERY task of fwd1,
    inv1 and the MAC runs its fix-up code (normally 2^-32 per element); results must not change.  Runs in a fresh
    process because the trigger is a __constant__ set when the context is created.  The throughput shape runs the
    FP64 step on the (integral) gate key unless NUFHE_B200_FFT=0 keeps its NTT step, which has the fix-up code.  Besides
    the gate, the script runs the separately compiled LUT instantiations (L = 2 with per-ciphertext test vectors, and a
    GLWE test vector) and extract2 with distinct job operands at an odd job batch, at n = 25 against the oracle."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, NUFHE_B200_FORCE_RARE_PATH='1')
    env['NUFHE_B200_FFT'] = '0' if wide_max == 'throughput_ntt' else '1'
    env['NUFHE_B200_PAIR_MAX'] = '1000000' if wide_max == 'pair' else '0'
    env.update({'NUFHE_B200_WIDE_MAX': '1000000', 'NUFHE_B200_WIDE2_MAX': '1000000'} if wide_max == 'wide2' else
               {'NUFHE_B200_WIDE_MAX': '1000000' if wide_max == '1000000' else '0', 'NUFHE_B200_WIDE2_MAX': '0'})
    r = subprocess.run([sys.executable, '-c', _RARE_PATH_SCRIPT % {'root': root}], env=env, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0 and 'rare path ok' in r.stdout, r.stdout + r.stderr
