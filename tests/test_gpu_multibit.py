"""Multi-bit bootstrap keys on the GPU (DESIGN.md section 14): every fused entry point bit for bit against the
multi-bit reference (tests/multibit_ref.py), the noiseless-key identity, and the Python API end to end."""
import numpy
import pytest
import torch

import multibit_ref as M
from oracle import oracle as O

pytestmark = pytest.mark.gpu

N = 1024
SEED = 20261016


@pytest.fixture(scope='module')
def eng():
    from nufhe_b200.engine import Engine
    return Engine()


@pytest.fixture(scope='module')
def keys():
    return O.OracleKeys(SEED)


@pytest.fixture(scope='module')
def mbkey(eng, keys):
    raw, ref = M.multibit_key(keys, SEED + 1)
    return raw, eng.bk_prepare_multibit(eng.to_device(ref))


def _dev(eng, x):
    return tuple(eng.to_device(numpy.ascontiguousarray(v)) for v in x)


def _host(eng, x):
    return tuple(eng.to_host(v) for v in x)


def _equal(got, want):
    return all(numpy.array_equal(numpy.asarray(g).reshape(numpy.asarray(w).shape), w) for g, w in zip(got, want))


def _inputs(keys, rng, B):
    return keys.encrypt(rng.randint(0, 2, B).astype(bool)), keys.encrypt(rng.randint(0, 2, B).astype(bool))


@pytest.mark.parametrize('B', [1, 2, 3, 64, 257, 4096])
def test_gate_bootstrap_matches_reference(eng, keys, mbkey, B):
    """nb_bootstrap_extract (gate_nand's prologue).  On a 132-SM H100 batches up to 528 are one wave of the 2-ciphertext
    shape; 4096 (every output compared) runs the chunked queue with parked accumulators."""
    raw, bk = mbkey
    rng = numpy.random.RandomState(B)
    x1, x2 = _inputs(keys, rng, B)
    num, den, sa, sb = O.GATE_TABLE['nand']
    c = O.phase_to_t32(num, den)
    got = _host(eng, eng.bootstrap_extract(_dev(eng, x1), _dev(eng, x2), c, sa, sb, O.MU, bk))
    want = M.bootstrap_extract(x1, x2, c, sa, sb, O.MU, raw, device='cuda')
    assert _equal(got, want)
    # and the gate's truth table after the key switch
    ra, rb, _ = eng.keyswitch(tuple(eng.to_device(v) for v in keys.ks), eng.bootstrap_extract(
        _dev(eng, x1), _dev(eng, x2), c, sa, sb, O.MU, bk))
    bits = keys.decrypt((eng.to_host(ra), eng.to_host(rb)))
    assert (bits == ~(keys.decrypt(x1) & keys.decrypt(x2))).all()


@pytest.mark.parametrize('B', [1, 2, 3, 64, 257, 1024])
def test_mux_pair_matches_reference(eng, keys, mbkey, B):
    """nb_bootstrap_extract2: gate_mux's two bootstraps in one launch; 1024 (2048 ciphertexts) runs the chunked queue"""
    raw, bk = mbkey
    rng = numpy.random.RandomState(100 + B)
    a, b = _inputs(keys, rng, B)
    c3 = keys.encrypt(rng.randint(0, 2, B).astype(bool))
    and_c = O.phase_to_t32(-1, 8)
    job_a, job_b = (a, b, and_c, 1, 1), (a, c3, and_c, -1, 1)
    ra, rb = eng.bootstrap_extract2(
        (_dev(eng, a), _dev(eng, b), and_c, 1, 1), (_dev(eng, a), _dev(eng, c3), and_c, -1, 1), O.MU, bk)
    got = (numpy.concatenate([eng.to_host(ra[0]), eng.to_host(rb[0])]), numpy.concatenate([eng.to_host(ra[1]), eng.to_host(rb[1])]))
    want = M.bootstrap_extract2(job_a, job_b, O.MU, raw, device='cuda')
    assert _equal(got, want)


@pytest.mark.parametrize('L,B,per_ct', [(0, 1, False), (0, 2, True), (0, 257, True), (0, 1024, True), (1, 3, False),
                                         (1, 64, False), (1, 1024, False), (2, 3, True), (2, 64, False),
                                         (2, 1024, True)])
def test_lut_bootstrap_matches_reference(eng, keys, mbkey, L, B, per_ct):
    """nb_bootstrap_lut_extract at L = 0, 1, 2, one test vector or one per ciphertext; 1024 runs the chunked queue"""
    raw, bk = mbkey
    rng = numpy.random.RandomState(200 + B + L)
    x1, x2 = _inputs(keys, rng, B)
    tv = rng.randint(-2**31, 2**31, size=(B, N) if per_ct else (N,), dtype=numpy.int64).astype(numpy.int32)
    got = _host(eng, eng.bootstrap_lut_extract(_dev(eng, x1), _dev(eng, x2), 0, 1, 2, eng.to_device(tv), L, bk))
    want = M.bootstrap_lut_extract(x1, x2, 0, 1, 2, tv, L, raw, device='cuda')
    assert _equal(got, want)


@pytest.mark.parametrize('B', [1, 2, 3, 64, 257, 1024])
def test_glwe_lut_bootstrap_matches_reference(eng, keys, mbkey, B):
    """nb_bootstrap_glwe_lut_extract: one GLWE test vector per ciphertext; 1024 runs the chunked queue"""
    raw, bk = mbkey
    rng = numpy.random.RandomState(300 + B)
    x, _ = _inputs(keys, rng, B)
    tv = rng.randint(-2**31, 2**31, size=(B, 2, N), dtype=numpy.int64).astype(numpy.int32)
    got = _host(eng, eng.bootstrap_glwe_lut_extract(_dev(eng, x), eng.to_device(tv), bk))
    want = M.bootstrap_glwe_lut_extract(x, tv, raw, device='cuda')
    assert _equal(got, want)


def test_noiseless_identity(eng, keys):
    """With noiseless keys and a test vector of multiples of 2^12 the rotation is exact: the GPU's multi-bit bootstrap
    extracts coefficient 0 of X^(sum abar_i s_i - barb) tv, with a zero mask"""
    raw, ref = M.multibit_key(keys, 0, noiseless=True)
    bk = eng.bk_prepare_multibit(eng.to_device(ref))
    rng = numpy.random.RandomState(5)
    B = 300
    a = rng.randint(-2**31, 2**31, size=(B, keys.n), dtype=numpy.int64).astype(numpy.int32)
    a[0] = 0
    a[1] = -2**31                                            # abar = N everywhere
    b = rng.randint(-2**31, 2**31, size=B, dtype=numpy.int64).astype(numpy.int32)
    tv = numpy.zeros((B, 2, N), numpy.int32)
    tv[:, 1] = (rng.randint(0, 2**20, size=(B, N)) << 12).astype(numpy.uint32).view(numpy.int32)
    ga, gb = _host(eng, eng.bootstrap_glwe_lut_extract(_dev(eng, (a, b)), eng.to_device(tv), bk))
    barb, bara = O.t32_to_phase(b, 2 * N), O.t32_to_phase(a, 2 * N)
    e = (bara.astype(numpy.int64) * keys.lwe_key).sum(-1) - barb
    assert (bara[1] == N).all()
    assert (ga == 0).all()
    assert numpy.array_equal(gb.reshape(B), M.exact_rotation(tv[:, 1], e)[:, 0])


def test_per_bit_entry_points_refuse_a_multibit_key(eng, keys, mbkey):
    _, bk = mbkey
    acc = eng.to_device(numpy.zeros((2, 2, N), numpy.int32))
    bara = eng.to_device(numpy.zeros((2, keys.n), numpy.int32))
    with pytest.raises(Exception, match='multi-bit'):
        eng.blind_rotate(acc, bara, bk)
    with pytest.raises(Exception, match='multi-bit'):
        eng.external_product(acc, bk, 0)


# ---- the Python API -------------------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def api():
    import nufhe_b200 as nufhe
    ctx = nufhe.Context(rng=nufhe.DeterministicRNG(SEED))
    sk = ctx.make_secret_key()
    ck = ctx.make_cloud_key(sk, multi_bit=2)
    return nufhe, ctx, sk, ck


def test_vm_gates_truth_tables_at_4096(api):
    nufhe, ctx, sk, ck = api
    assert isinstance(ck.bootstrap_key, nufhe.MultiBitBootstrapKey)
    vm = ctx.make_virtual_machine(ck)
    rng = numpy.random.RandomState(7)
    a, b, c = (rng.randint(0, 2, 4096).astype(bool) for _ in range(3))
    ca, cb, cc = (ctx.encrypt(sk, x) for x in (a, b, c))
    for name, f in (('nand', lambda x, y: ~(x & y)), ('and', lambda x, y: x & y), ('or', lambda x, y: x | y),
                    ('xor', lambda x, y: x ^ y), ('xnor', lambda x, y: ~(x ^ y)), ('nor', lambda x, y: ~(x | y)),
                    ('andny', lambda x, y: ~x & y), ('andyn', lambda x, y: x & ~y), ('orny', lambda x, y: ~x | y),
                    ('oryn', lambda x, y: x | ~y)):
        assert (ctx.decrypt(sk, getattr(vm, 'gate_' + name)(ca, cb)) == f(a, b)).all(), name
    assert (ctx.decrypt(sk, vm.gate_mux(ca, cb, cc)) == numpy.where(a, b, c)).all()
    assert (ctx.decrypt(sk, vm.gate_not(ca)) == ~a).all()


def test_vm_luts_at_allowed_configurations(api):
    nufhe, ctx, sk, ck = api
    vm = ctx.make_virtual_machine(ck)
    rng = numpy.random.RandomState(8)
    x = rng.randint(0, 4, 1024)
    cx = ctx.encrypt_int(sk, x, 2)
    sq = vm.make_lut([(v * v) % 4 for v in range(4)], 2)
    assert (ctx.decrypt_int(sk, vm.lut(sq, cx), 2) == (x * x) % 4).all()
    y = rng.randint(0, 2, 1024)
    cy = ctx.encrypt_int(sk, y, 1)
    t2 = vm.make_lut([[v & 1 for v in range(2)], [1 - (v & 1) for v in range(2)]], 1)
    r0, r1 = vm.lut(t2, cy)
    assert (ctx.decrypt_int(sk, r0, 1) == y).all() and (ctx.decrypt_int(sk, r1, 1) == 1 - y).all()


def test_compressed_tree_key_and_packed_outputs(api):
    nufhe, ctx, sk, _ = api
    cck, tree_key = ctx.make_cloud_key(sk, compressed=True, tree_key=True, multi_bit=2)
    ck = cck.decompress(ctx.thread)
    assert isinstance(ck.bootstrap_key, nufhe.MultiBitBootstrapKey)
    vm = ctx.make_virtual_machine(ck)
    rng = numpy.random.RandomState(9)
    a, b = (rng.randint(0, 2, 512).astype(bool) for _ in range(2))
    r = vm.gate_nand(ctx.encrypt(sk, a), ctx.encrypt(sk, b))
    psk, pk = ctx.make_packing_keys(sk)
    assert (ctx.decrypt(psk, vm.pack(pk, r)) == ~(a & b)).all()
    d1, d0 = rng.randint(0, 2, 256), rng.randint(0, 2, 256)
    table = vm.make_tree_lut(numpy.array([[0, 1], [1, 0]]), 1, 2)
    t = vm.lut_tree(tree_key, table, [ctx.encrypt_int(sk, d1, 1), ctx.encrypt_int(sk, d0, 1)])
    assert (ctx.decrypt_int(sk, t, 1) == d1 ^ d0).all()


def test_uint_min_capture_is_bit_identical(api):
    nufhe, ctx, sk, ck = api
    from nufhe_b200.operators_integer import uint_min
    vm = ctx.make_virtual_machine(ck)
    rng = numpy.random.RandomState(10)
    shape, bits = (64,), 4
    x = rng.randint(0, 2, shape + (bits,)).astype(bool)
    y = rng.randint(0, 2, shape + (bits,)).astype(bool)
    cx, cy = ctx.encrypt(sk, x), ctx.encrypt(sk, y)
    eager = vm.empty_ciphertext(shape + (bits,))
    uint_min(ctx.thread, ck, eager, cx, cy)
    out = vm.empty_ciphertext(shape + (bits,))
    graph = vm.capture(lambda: uint_min(ctx.thread, ck, out, cx, cy))
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out.a, eager.a) and torch.equal(out.b, eager.b)
    w = 1 << numpy.arange(bits)[::-1]                      # big-endian bits (operators_integer.uint_min)
    xv = (x * w).sum(-1)
    yv = (y * w).sum(-1)
    got = (ctx.decrypt(sk, out) * w).sum(-1)
    assert (got == numpy.minimum(xv, yv)).all()


def test_output_noise_matches_the_estimate(api):
    """65 536 bootstraps of fresh encryptions through an identity table (P = 1): variance of the output phase error
    within 0.5 - 2x the estimate (nufhe_b200/lut.py: multi-bit rules), no error beyond 7 sigma"""
    nufhe, ctx, sk, ck = api
    from nufhe_b200.lut import bootstrap_variance
    vm = ctx.make_virtual_machine(ck)
    rng = numpy.random.RandomState(11)
    x = rng.randint(0, 2, 65536)
    ident = vm.make_lut([0, 1], 1)
    r = vm.lut(ident, ctx.encrypt_int(sk, x, 1))
    from nufhe_b200.lwe import lwe_decrypt
    ph = numpy.asarray(lwe_decrypt(ctx.thread, r, sk.lwe_key)).astype(numpy.int64)
    want = (x << 30).astype(numpy.int64)
    err = (((ph - want) + 2**31) % 2**32 - 2**31) / 2**32
    est = bootstrap_variance(ck.params, multi_bit=2)
    ratio = err.var() / est
    print('multi-bit output variance %.3e, estimate %.3e, ratio %.2f, max |err| %.4f' % (err.var(), est, ratio,
                                                                                          abs(err).max()))
    assert 0.5 <= ratio <= 2
    assert abs(err).max() < 7 * numpy.sqrt(est)
