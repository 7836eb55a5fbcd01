"""Tree-based programmable bootstrapping on the GPU: nb_tree_keyswitch and nb_tree_assemble bit for bit against the
NumPy restatement (tree_ref.py), nb_bootstrap_glwe_lut_extract against nb_bootstrap_lut_extract and against the
separate steps in every CTA shape, and vm.lut_tree end to end, with its noise."""
import numpy
import pytest
import torch

import nufhe_b200
from nufhe_b200 import lut, tree_lut
from nufhe_b200.random_numbers import DeterministicRNG
import gen_inputs as G
from oracle import oracle as O
import tree_ref

pytestmark = pytest.mark.gpu
N = 1024


@pytest.fixture(scope='module')
def eng():
    from nufhe_b200.engine import Engine
    return Engine()


@pytest.fixture(scope='module')
def bk_int(eng):
    return eng.bk_prepare(eng.to_device(O.OracleKeys(G.GATE_SEED).bk))


def _rand(rng, shape):
    return rng.randint(-2**31, 2**31, size=shape, dtype=numpy.int64).astype(numpy.int32)


@pytest.mark.parametrize('rows,k', [(1, 1), (17, 1), (129, 2), (4096, 1)])
def test_keyswitch_matches_restatement(eng, rows, k):
    rng = numpy.random.RandomState(rows + k)
    n = 500
    a = _rand(rng, (rows, n))
    masks, body = _rand(rng, (n, 2, k, N)), _rand(rng, (n, 2, N))
    planes = eng.tree_prepare(eng.to_device(masks), eng.to_device(body))
    got = eng.to_host(eng.tree_keyswitch(eng.to_device(a), planes, k))
    assert (got == tree_ref.keyswitch(a, masks, body)).all()


def test_keyswitch_at_the_exactness_bound(eng):
    n = 500
    a = numpy.full((64, n), 0x7f7f8000, numpy.int64).astype(numpy.int32)       # every digit -128
    masks = numpy.full((n, 2, 1, N), -2**31, numpy.int32)
    body = numpy.full((n, 2, N), -2**31, numpy.int32)
    masks[:, :, :, 1::2] = 2**31 - 1
    body[:, :, ::3] = 1
    planes = eng.tree_prepare(eng.to_device(masks), eng.to_device(body))
    got = eng.to_host(eng.tree_keyswitch(eng.to_device(a), planes, 1))
    assert (got == tree_ref.keyswitch(a, masks, body)).all()


@pytest.mark.parametrize('bits', [1, 2])
@pytest.mark.parametrize('k', [1, 2])
def test_assemble_matches_restatement(eng, bits, k):
    rng = numpy.random.RandomState(10 * bits + k)
    T, M = 37, 1 << bits
    v, b = _rand(rng, (T, M, k + 1, N)), _rand(rng, (T, M))
    got = eng.to_host(eng.tree_assemble(eng.to_device(v), eng.to_device(b), bits))
    assert (got == tree_ref.assemble(v, b, bits)).all()


def test_bad_arguments_are_rejected(eng, bk_int):
    z = torch.zeros(16, dtype=torch.int32, device=eng.device)
    p = z.data_ptr()
    with pytest.raises(ValueError, match='null'):
        eng._call('nb_tree_keyswitch', None, p, 500, 1, p, 4)
    with pytest.raises(ValueError):
        eng._call('nb_tree_keyswitch', p, p, 70000, 1, p, 4)                   # past the exactness bound
    with pytest.raises(ValueError):
        eng._call('nb_tree_assemble', p, p, 3, 1, p, 4)
    with pytest.raises(ValueError, match='null'):
        eng._call('nb_tree_prepare', p, None, 500, 1, p)
    with pytest.raises(ValueError, match='null'):
        eng._call('nb_bootstrap_glwe_lut_extract', p, p, None, bk_int.data_ptr(), 500, p, p, 4)
    eng._call('nb_tree_keyswitch', p, p, 500, 1, p, 0)                          # batch 0: a no-op
    eng._call('nb_tree_assemble', p, p, 2, 1, p, 0)
    eng._call('nb_bootstrap_glwe_lut_extract', p, p, p, bk_int.data_ptr(), 500, p, p, 0)


@pytest.mark.parametrize('B', [1, 16, 64, 256, 4096])
def test_trivial_glwe_test_vector_equals_the_lut_kernel(eng, bk_int, B):
    """Zero masks and body = a plaintext test vector: the same bits as nb_bootstrap_lut_extract (tv_stride 1024); the
    batches select every CTA shape."""
    rng = numpy.random.RandomState(B)
    a, b = _rand(rng, (B, 500)), _rand(rng, (B,))
    tv = _rand(rng, (B, N))
    x = (eng.to_device(a), eng.to_device(b))
    want = eng.bootstrap_lut_extract(x, None, 0, 1, 0, eng.to_device(tv), 0, bk_int)
    glwe = numpy.zeros((B, 2, N), numpy.int32)
    glwe[:, 1] = tv
    got = eng.bootstrap_glwe_lut_extract(x, eng.to_device(glwe), bk_int)
    assert torch.equal(want[0], got[0]) and torch.equal(want[1], got[1])


@pytest.mark.parametrize('B', [1, 64, 4096])
def test_encrypted_test_vector_equals_the_steps(eng, bk_int, B):
    """A random GLWE tv: the same bits as t32_to_phase, nb_shift_torus_polynomial of both polynomials and
    nb_blind_rotate with that explicit accumulator."""
    rng = numpy.random.RandomState(100 + B)
    a, b = _rand(rng, (B, 500)), _rand(rng, (B,))
    tv = eng.to_device(_rand(rng, (B, 2, N)))
    x = (eng.to_device(a), eng.to_device(b))
    got = eng.bootstrap_glwe_lut_extract(x, tv, bk_int)
    barb, bara = torch.empty_like(x[1]), torch.empty_like(x[0])
    eng.t32_to_phase(barb, x[1], 2 * N)
    eng.t32_to_phase(bara, x[0], 2 * N)
    acc = torch.empty((B, 2, N), dtype=torch.int32, device=eng.device)
    eng.shift_torus_polynomial(acc, tv, barb, polys_per_power=2, mode=eng.SHIFT_INVERT)
    wa, wb, _ = eng.blind_rotate(acc, bara, bk_int)
    assert torch.equal(wa, got[0]) and torch.equal(wb, got[1])


# ---------------------------------------------------------------- end to end

def _setup(seed, k=1, compressed=False):
    ctx = nufhe_b200.Context(rng=DeterministicRNG(seed))
    sk = ctx.make_secret_key(tlwe_mask_size=k)
    ck, tk = ctx.make_cloud_key(sk, compressed=compressed, tree_key=True)
    if compressed:
        ck = ck.decompress(ctx.thread)
    return ctx, sk, ck, tk


@pytest.fixture(scope='module')
def keys():
    return _setup(81)


def _digits(rng, bits, D, B):
    return [rng.randint(0, 1 << bits, size=B) for _ in range(D)]        # d_{D-1}, ..., d_0


@pytest.mark.parametrize('bits,D,F,B', [(2, 2, 1, 4096), (2, 2, 2, 4096), (2, 3, 1, 4096), (1, 4, 1, 4096),
                                        (2, 4, 1, 64)])
def test_lut_tree_decrypts_exactly(keys, bits, D, F, B):
    ctx, sk, ck, tk = keys
    vm = ctx.make_virtual_machine(ck)
    rng = numpy.random.RandomState(bits * 100 + D * 10 + F)
    M = 1 << bits
    tables = rng.randint(0, M, size=((F,) if F > 1 else ()) + (M,) * D)
    values = _digits(rng, bits, D, B)
    if B >= M**D:        # every combination at least once
        grid = numpy.stack(numpy.meshgrid(*[numpy.arange(M)] * D, indexing='ij'), -1).reshape(-1, D)
        for i in range(D):
            values[i][:grid.shape[0]] = grid[:, i]
    out = vm.lut_tree(tk, vm.make_tree_lut(tables, bits, D), [ctx.encrypt_int(sk, v, bits) for v in values])
    out = out if F > 1 else [out]
    want = tables[(slice(None),) + tuple(values)] if F > 1 else tables[tuple(values)][None]
    for f in range(F):
        assert (ctx.decrypt_int(sk, out[f], bits) == want[f]).all(), f


def test_lut_tree_compressed_key_public_key_and_bool(keys):
    ctx, sk, ck, tk = _setup(82, compressed=True)
    vm = ctx.make_virtual_machine(ck)
    pub = ctx.make_public_key(sk)
    rng = numpy.random.RandomState(5)
    B = 1024
    x, y = rng.randint(0, 4, B), rng.randint(0, 4, B)
    cx, cy = ctx.encrypt_int(pub, x, 2), ctx.encrypt_int(pub, y, 2)
    less = vm.make_tree_lut(numpy.less.outer(numpy.arange(4), numpy.arange(4)), 2, 2, out='bool')
    lt = vm.lut_tree(tk, less, [cx, cy])
    assert (ctx.decrypt(sk, lt) == (x < y)).all()
    # bool outputs feed the gates: NOT(x < y AND y < x) is always true
    gt = vm.lut_tree(tk, less, [cy, cx])
    assert (ctx.decrypt(sk, vm.gate_nand(lt, gt)) == True).all()       # noqa: E712
    prod = vm.lut_tree(tk, vm.make_tree_lut(numpy.multiply.outer(numpy.arange(4), numpy.arange(4)) % 4, 2, 2),
                       [cx, cy])
    assert (ctx.decrypt_int(sk, prod, 2) == (x * y) % 4).all()


def test_lut_tree_capture(keys):
    """vm.capture records lut_tree with table.reserve_batch(B) reserved; the replay gives the eager results."""
    ctx, sk, ck, tk = keys
    vm = ctx.make_virtual_machine(ck)
    rng = numpy.random.RandomState(8)
    B = 300
    table = rng.randint(0, 4, size=(4, 4))
    x, y = rng.randint(0, 4, B), rng.randint(0, 4, B)
    cx, cy = ctx.encrypt_int(sk, x, 2), ctx.encrypt_int(sk, y, 2)
    t = vm.make_tree_lut(table, 2, 2)
    eager = vm.lut_tree(tk, t, [cx, cy])
    g = vm.capture(lambda: vm.lut_tree(tk, t, [cx, cy]), reserve_batch=t.reserve_batch(B))
    out = g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out.a, eager.a) and torch.equal(out.b, eager.b)
    assert (ctx.decrypt_int(sk, out, 2) == table[x, y]).all()


def test_lut_tree_mask_size_2():
    ctx, sk, ck, tk = _setup(83, k=2)
    vm = ctx.make_virtual_machine(ck)
    rng = numpy.random.RandomState(6)
    x, y = rng.randint(0, 4, 8), rng.randint(0, 4, 8)
    table = rng.randint(0, 4, size=(4, 4))
    r = vm.lut_tree(tk, vm.make_tree_lut(table, 2, 2), [ctx.encrypt_int(sk, x, 2), ctx.encrypt_int(sk, y, 2)])
    assert (ctx.decrypt_int(sk, r, 2) == table[x, y]).all()


def test_lut_tree_noise(keys):
    """65 536 level-2 outputs at P = 2: the sample variance of the output phase error is 0.5 - 2 times the estimate
    (tree_lut.output_variance) and no error lies beyond 7 standard deviations."""
    ctx, sk, ck, tk = keys
    vm = ctx.make_virtual_machine(ck)
    rng = numpy.random.RandomState(9)
    B = 65536
    table = rng.randint(0, 4, size=(4, 4))
    x, y = rng.randint(0, 4, B), rng.randint(0, 4, B)
    r = vm.lut_tree(tk, vm.make_tree_lut(table, 2, 2), [ctx.encrypt_int(sk, x, 2), ctx.encrypt_int(sk, y, 2)])
    key = sk.lwe_key.key.to(torch.int64)
    phase = (r.b.to(torch.int64) - (r.a.to(torch.int64) * key).sum(-1)) & 0xffffffff
    err = ((phase.cpu().numpy() - lut.encode_int(table[x, y], 2).astype(numpy.int64) + 2**31) % 2**32 - 2**31) / 2**32
    est = tree_lut.output_variance(sk.params, 2, 2)
    assert 0.5 * est < err.var() < 2 * est, (err.var(), est)
    assert numpy.abs(err).max() < 7 * est**0.5
