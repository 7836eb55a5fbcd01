"""Programmable bootstrapping on the GPU: nb_bootstrap_lut_extract against the gate path and the oracle's composition
of the reference's steps, and lookup tables end to end through the VirtualMachine."""
import numpy
import pytest
import torch

import gen_inputs as G
from oracle import oracle as O
from fused_ref import oracle_lut

pytestmark = pytest.mark.gpu
N = 1024


@pytest.fixture(scope='module')
def eng():
    from nufhe_b200.engine import Engine
    return Engine()


@pytest.fixture(scope='module')
def keys():
    return O.OracleKeys(G.GATE_SEED)


@pytest.fixture(scope='module')
def dev_keys(eng, keys):
    return eng.bk_prepare(eng.to_device(keys.bk)), tuple(eng.to_device(x) for x in keys.ks)


def _random_lwe(rng, B):
    return (rng.randint(-2**31, 2**31, size=(B, O.LWE_N), dtype=numpy.int64).astype(numpy.int32),
            rng.randint(-2**31, 2**31, size=B, dtype=numpy.int64).astype(numpy.int32))


def _dev(eng, x):
    return (eng.to_device(x[0]), eng.to_device(x[1]))


def test_constant_test_vector_equals_the_gate_path(eng, keys, dev_keys):
    bk_int, _ = dev_keys
    rng = G.rs(900)
    B = 4096
    a, b = (keys.encrypt(rng.randint(0, 2, B).astype(bool)) for _ in range(2))
    num, den, sa, sb = O.GATE_TABLE['nand']
    c = O.phase_to_t32(num, den)
    gate = eng.bootstrap_extract(_dev(eng, a), _dev(eng, b), c, sa, sb, O.MU, bk_int)
    tv = eng.to_device(numpy.full(N, O.MU, numpy.int32))
    got = eng.bootstrap_lut_extract(_dev(eng, a), _dev(eng, b), c, sa, sb, tv, 0, bk_int)
    assert torch.equal(gate[0], got[0]) and torch.equal(gate[1], got[1])


@pytest.mark.parametrize('L', [0, 1, 2])
@pytest.mark.parametrize('per_ct', [False, True])
def test_random_test_vectors_match_the_oracle(eng, keys, dev_keys, L, per_ct):
    """B = 4096 on the GPU; the oracle recomputes every output of 48 ciphertexts spread over the batch (its 500-step
    rotation takes about 0.1 s per ciphertext on the CPU).  Bivariate prologue x1 * 2 + x2 with a constant."""
    bk_int, _ = dev_keys
    rng = G.rs(910 + 2 * L + per_ct)
    B, K = 4096, 1 << L
    x1, x2 = _random_lwe(rng, B), _random_lwe(rng, B)
    tv = rng.randint(-2**31, 2**31, size=(B, N) if per_ct else (N,), dtype=numpy.int64).astype(numpy.int32)
    c = 12345678
    ga, gb = eng.bootstrap_lut_extract(_dev(eng, x1), _dev(eng, x2), c, 2, 1, eng.to_device(tv), L, bk_int)
    assert ga.shape == (B * K, N) and gb.shape == (B * K,)
    ga, gb = eng.to_host(ga).reshape(B, K, N), eng.to_host(gb).reshape(B, K)
    pick = numpy.sort(rng.choice(B, 48, replace=False))
    pick[0], pick[-1] = 0, B - 1
    with numpy.errstate(over='ignore'):
        xa = (2 * x1[0][pick] + x2[0][pick]).astype(numpy.int32)
        xb = (c + 2 * x1[1][pick] + x2[1][pick]).astype(numpy.int32)
    wa, wb = oracle_lut(xa, xb, tv[pick] if per_ct else tv, L, keys.bk)
    assert (ga[pick].reshape(-1, N) == wa).all() and (gb[pick].reshape(-1) == wb).all()


def test_bad_arguments_are_rejected(eng, dev_keys):
    bk_int, _ = dev_keys
    x = (torch.zeros((2, O.LWE_N), dtype=torch.int32, device=eng.device), torch.zeros(2, dtype=torch.int32, device=eng.device))
    tv = torch.zeros(N, dtype=torch.int32, device=eng.device)
    with pytest.raises(ValueError):
        eng.bootstrap_lut_extract(x, None, 0, 1, 0, tv, 3, bk_int)
    with pytest.raises(ValueError, match='null'):
        eng._call('nb_bootstrap_lut_extract', x[0].data_ptr(), x[1].data_ptr(), None, None, 0, 1, 0, None, 0, 0,
                  bk_int.data_ptr(), O.LWE_N, x[0].data_ptr(), x[1].data_ptr(), 2)
    with pytest.raises(ValueError, match='stride'):
        eng._call('nb_bootstrap_lut_extract', x[0].data_ptr(), x[1].data_ptr(), None, None, 0, 1, 0, tv.data_ptr(), 512,
                  0, bk_int.data_ptr(), O.LWE_N, x[0].data_ptr(), x[1].data_ptr(), 2)


@pytest.fixture(scope='module')
def api():
    import nufhe_b200
    ctx = nufhe_b200.Context(rng=nufhe_b200.DeterministicRNG(4242))
    sk, ck = ctx.make_key_pair()
    return nufhe_b200, ctx, sk, ck, ctx.make_virtual_machine(ck)


def test_fused_path_equals_the_separate_steps(api):
    nufhe, ctx, sk, ck, vm = api
    vm_steps = ctx.make_virtual_machine(ck, perf_params=nufhe.PerformanceParameters(ck.params, single_kernel_bootstrap=False))
    rng = numpy.random.RandomState(5)
    x, y = ctx.encrypt_int(sk, rng.randint(0, 2, 64), 2), ctx.encrypt_int(sk, rng.randint(0, 2, 64), 2)
    for table, args in ((vm.make_lut([[0, 1, 0, 1], [0, 0, 1, 1]], 2), (x,)),
                        (vm.make_lut(rng.randint(0, 4, (64, 4)), 2, log2_outputs=0), (x,)),
                        (vm.make_lut([3, 1, 2, 0], 2), (x, y, 0)),
                        (vm.make_lut(numpy.zeros((4, 2)) + [0, 1], 1), (x,))):
        fused, steps = vm.lut(table, *args), vm_steps.lut(table, *args)
        for f, s in zip(fused if isinstance(fused, list) else [fused], steps if isinstance(steps, list) else [steps]):
            assert torch.equal(f.a, s.a) and torch.equal(f.b, s.b)


EVALS = 65536


def _fresh_lut_outputs(ctx, sk, vm, values, bits):
    """Inputs that carry a LUT output's noise: fresh encryptions through the identity table."""
    return vm.lut(vm.make_lut(list(range(2**bits)), bits), ctx.encrypt_int(sk, values, bits))


def test_tables_decrypt_exactly(api):
    """Identity, negation, square, constant and random tables at P = 1, 2 (L = 0), over 65 536 inputs each; P = 3 is
    refused (6.7 sigma of measured margin)."""
    nufhe, ctx, sk, ck, vm = api
    rng = numpy.random.RandomState(11)
    with pytest.raises(ValueError):
        vm.lut(vm.make_lut(list(range(8)), 3), ctx.encrypt_int(sk, [0, 1], 3))
    for bits in (1, 2):
        M = 2**bits
        m = rng.randint(0, M, EVALS)
        x = _fresh_lut_outputs(ctx, sk, vm, m, bits)
        for f in (numpy.arange(M), (-numpy.arange(M)) % M, numpy.arange(M)**2 % M, numpy.full(M, M - 1),
                  rng.randint(0, M, M)):
            got = ctx.decrypt_int(sk, vm.lut(vm.make_lut(f, bits), x), bits)
            assert (got == f[m]).all(), (bits, f, int((got != f[m]).sum()))
        bool_out = vm.lut(vm.make_lut(numpy.arange(M) % 2, bits, out='bool'), x)
        assert (ctx.decrypt(sk, bool_out) == (m % 2 == 1)).all()


def test_many_outputs_and_bivariate_decrypt_exactly(api):
    nufhe, ctx, sk, ck, vm = api
    rng = numpy.random.RandomState(12)
    # P = 1, L = 2: four functions of one bit
    m = rng.randint(0, 2, EVALS)
    x = _fresh_lut_outputs(ctx, sk, vm, m, 1)
    fs = numpy.array([[0, 1], [1, 0], [1, 1], [0, 0]])
    for f, r in zip(fs, vm.lut(vm.make_lut(fs, 1), x)):
        assert (ctx.decrypt_int(sk, r, 1) == f[m]).all()
    # P = 2, bivariate x + y (shift 0) at L = 1 and L = 0
    a, b = rng.randint(0, 2, EVALS), rng.randint(0, 2, EVALS)
    xa, xb = _fresh_lut_outputs(ctx, sk, vm, a, 2), _fresh_lut_outputs(ctx, sk, vm, b, 2)
    s, c = vm.lut(vm.make_lut([[0, 1, 0, 1], [0, 0, 1, 1]], 2), xa, xb)
    assert (ctx.decrypt_int(sk, s, 2) == (a + b) % 2).all() and (ctx.decrypt_int(sk, c, 2) == (a + b) // 2).all()
    f = numpy.array([2, 3, 0, 1])
    r = vm.lut(vm.make_lut(f, 2), xa, xb)
    assert (ctx.decrypt_int(sk, r, 2) == f[a + b]).all()
    with pytest.raises(ValueError):
        vm.lut(vm.make_lut(f, 2), xa, xb, shift=1)


def test_full_adder_and_chain(api):
    nufhe, ctx, sk, ck, vm = api
    rng = numpy.random.RandomState(13)
    # the full adder over all 8 inputs, 8192 times each: sum and carry from one two-output bootstrap
    bits = rng.randint(0, 2, (3, EVALS))
    bits[:, :8] = numpy.array([[i >> k & 1 for i in range(8)] for k in range(3)])
    ins = [_fresh_lut_outputs(ctx, sk, vm, v, 2) for v in bits]
    adder = vm.make_lut([[0, 1, 0, 1], [0, 0, 1, 1]], 2)
    s, c = vm.lut(adder, vm.int_add(vm.int_add(ins[0], ins[1]), ins[2]))
    total = bits.sum(0)
    assert (ctx.decrypt_int(sk, s, 2) == total % 2).all() and (ctx.decrypt_int(sk, c, 2) == total // 2).all()
    # a chain of 16 LUTs (x -> 3x + 1 mod 4)
    m = rng.randint(0, 4, 4096)
    x = ctx.encrypt_int(sk, m, 2)
    step = vm.make_lut((3 * numpy.arange(4) + 1) % 4, 2)
    for _ in range(16):
        x = vm.lut(step, x)
        m = (3 * m + 1) % 4
    assert (ctx.decrypt_int(sk, x, 2) == m).all()


def test_mask_size_2_key_decrypts():
    import nufhe_b200
    ctx = nufhe_b200.Context(rng=nufhe_b200.DeterministicRNG(77))
    sk, ck = ctx.make_key_pair(tlwe_mask_size=2)
    vm = ctx.make_virtual_machine(ck)
    m = numpy.arange(32) % 4
    r = vm.lut(vm.make_lut([[1, 2, 3, 0], [0, 0, 1, 1]], 2), ctx.encrypt_int(sk, m, 2))
    assert (ctx.decrypt_int(sk, r[0], 2) == (m + 1) % 4).all() and (ctx.decrypt_int(sk, r[1], 2) == m // 2).all()


def test_captured_lut_circuit_replays_bit_identical(api):
    nufhe, ctx, sk, ck, vm = api
    rng = numpy.random.RandomState(14)
    B = 512
    a, b = ctx.encrypt_int(sk, rng.randint(0, 2, B), 2), ctx.encrypt_int(sk, rng.randint(0, 2, B), 2)
    adder = vm.make_lut([[0, 1, 0, 1], [0, 0, 1, 1]], 2)
    neg = vm.make_lut([0, 3, 2, 1], 2)

    def circuit():
        s, c = vm.lut(adder, a, b)
        return vm.lut(neg, vm.int_add(s, c)), c

    eager = circuit()
    graph = vm.capture(circuit, reserve_batch=2 * B)
    replayed = graph.replay()
    torch.cuda.synchronize()
    for e, r in zip(eager, replayed):
        assert torch.equal(e.a, r.a) and torch.equal(e.b, r.b)
