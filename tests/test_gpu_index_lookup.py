"""Encrypted-index lookups on the GPU (DESIGN.md section 15): the three entry points bit for bit against the
oracle-composed reference (tests/index_ref.py), and vm.lookup end to end against the plaintext tables, into gates and
LUTs, with compressed selectors and a compressed multi-bit cloud key, and its output noise."""
import numpy
import pytest
import torch

import index_ref as R
from oracle import oracle as O

pytestmark = pytest.mark.gpu

N = 1024
GROUPS = 8                  # distinct selector sets; query q uses set q % GROUPS, so neighbouring CTA slots differ


@pytest.fixture(scope='module')
def eng():
    from nufhe_b200.engine import Engine
    return Engine(0)


def _rand_i32(rng, shape):
    return rng.randint(-2**31, 2**31, size=shape, dtype=numpy.int64).astype(numpy.int32)


def test_prepare_matches_bk_prepare(eng):
    """nb_index_prepare's spectra equal the FP64 part that nb_bk_prepare makes from the same rows in the reference form"""
    rng = numpy.random.RandomState(1)
    rows = _rand_i32(rng, (5, 2, 2, 2, N))
    rows[0] = -2**31
    rows[1] = 2**31 - 1
    spec = eng.to_host(eng.index_prepare(eng.to_device(rows)))
    bk = eng.to_host(eng.bk_prepare(eng.to_device(R.transform(rows))))
    ntt = eng.lib.nb_bk_row_u64() - eng.lib.nb_bk_multibit_row_u64()
    assert numpy.array_equal(spec, bk[:, ntt:])


def _case(eng, rng, Q, m, W):
    """random selector rows in GROUPS sets, a random table; (device selectors, reference rows, reference sets, polys)"""
    sets = _rand_i32(rng, (GROUPS, m, 2, 2, 2, N))
    q_set = numpy.arange(Q) % GROUPS
    sel = eng.to_device(sets)[torch.from_numpy(q_set).to(eng.device)]             # (Q, m, 2, 2, 2, N)
    ref = R.transform(sets)                                                         # row g m + j
    rows = q_set[:, None] * m + numpy.arange(m)[None, :]
    polys = R.table_polys(_rand_i32(rng, (W, 1 << m)), m)
    return sel, ref, rows, polys


@pytest.mark.parametrize('Q, m, W', [(1, 11, 1), (2, 11, 1), (3, 11, 1), (64, 11, 1), (257, 11, 1), (4096, 11, 1),
                                     (64, 1, 1), (64, 1, 512), (64, 8, 4), (64, 10, 3), (64, 16, 1), (3, 20, 1)])
def test_entry_points_match_reference(eng, Q, m, W):
    """every CMux level (nb_index_cmux_level, the first one on the shared plaintext level) and the rotation with
    extraction (nb_index_rotate_extract), bit for bit against the reference"""
    rng = numpy.random.RandomState(Q * 31 + m * 7 + W)
    sel, ref, rows, polys = _case(eng, rng, Q, m, W)
    spec = eng.index_prepare(sel).reshape(Q, m, -1)
    cur_d = eng.to_device(polys)
    cur = numpy.broadcast_to(polys, (Q,) + polys.shape).copy()
    for j in range(10, m):
        cur_d = eng.index_cmux_level(cur_d, spec, j, Q)
        if j < 12 or j == m - 1 or Q <= 3:
            cur = R.cmux_level(cur, ref, rows[:, j])
            assert numpy.array_equal(eng.to_host(cur_d), cur), 'level %d' % j
        else:
            cur = eng.to_host(cur_d)             # (the deep levels of m = 16 are checked from the GPU's input)
    a, b = eng.index_rotate_extract(cur_d, spec, m, W, Q)
    wa, wb = R.rotate_extract(cur, ref, rows, m, W)
    assert numpy.array_equal(eng.to_host(a), wa) and numpy.array_equal(eng.to_host(b), wb)


# ---- vm.lookup end to end --------------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def api():
    import nufhe_b200 as nufhe
    ctx = nufhe.Context(rng=nufhe.DeterministicRNG(2026))
    sk = ctx.make_secret_key()
    ck, ik = ctx.make_cloud_key(sk, index_key=True)
    vm = ctx.make_virtual_machine(ck)
    return nufhe, ctx, sk, ik, vm


@pytest.fixture(scope='module')
def idx16(api):
    nufhe, ctx, sk, ik, vm = api
    values = numpy.random.RandomState(16).randint(0, 1 << 16, size=4096)
    values[:2] = 0, (1 << 16) - 1
    return values, ctx.encrypt_index(ik, values, 16)


def test_lookup_m8_four_columns_into_lut(api):
    nufhe, ctx, sk, ik, vm = api
    rng = numpy.random.RandomState(8)
    values = rng.randint(0, 256, size=(64, 64))
    tab = rng.randint(0, 4, size=(4, 256))
    res = vm.lookup(ctx.encrypt_index(ik, values, 8), vm.make_index_table(tab, out='int', bits=2))
    assert len(res) == 4
    for w in range(4):
        assert res[w].shape == (64, 64)
        assert numpy.array_equal(ctx.decrypt_int(sk, res[w], 2), tab[w][values])
    f = vm.make_lut([3, 2, 1, 0], 2)
    assert numpy.array_equal(ctx.decrypt_int(sk, vm.lut(f, res[1]), 2), 3 - tab[1][values])


def test_lookup_m16_bool_into_gate_nand(api, idx16):
    nufhe, ctx, sk, ik, vm = api
    values, e = idx16
    tab = numpy.random.RandomState(17).randint(0, 2, size=(2, 1 << 16))
    r0, r1 = vm.lookup(e, vm.make_index_table(tab, out='bool'))
    assert numpy.array_equal(ctx.decrypt(sk, r0), tab[0][values].astype(bool))
    assert numpy.array_equal(ctx.decrypt(sk, r1), tab[1][values].astype(bool))
    assert numpy.array_equal(ctx.decrypt(sk, vm.gate_nand(r0, r1)), ~(tab[0][values] & tab[1][values]).astype(bool))


def test_several_passes_give_the_same_bits(api, monkeypatch):
    from nufhe_b200 import index_lookup as IL
    nufhe, ctx, sk, ik, vm = api
    rng = numpy.random.RandomState(12)
    values = rng.randint(0, 1 << 12, size=4096)
    raw = rng.randint(0, 4, size=1 << 12)
    tab = vm.make_index_table(raw, out='int', bits=2)
    e = ctx.encrypt_index(ik, values, 12)
    monkeypatch.setattr(IL, 'PASS_BYTES', 4096 * (12 * 2**17 + 4 * 8192))
    whole = vm.lookup(e, tab)
    monkeypatch.setattr(IL, 'PASS_BYTES', 700 * (12 * 2**17 + 4 * 8192))
    assert IL.queries_per_pass(12, 1) == 700
    parts = vm.lookup(e, tab)
    assert torch.equal(whole.a, parts.a) and torch.equal(whole.b, parts.b)
    assert numpy.array_equal(ctx.decrypt_int(sk, parts, 2), raw[values])


def test_compressed_selectors(api):
    nufhe, ctx, sk, ik, vm = api
    rng = numpy.random.RandomState(10)
    values = rng.randint(0, 1024, size=4096)
    tab = rng.randint(0, 8, size=1024)
    c = ctx.encrypt_index(ik, values, 10, compressed=True)
    table = vm.make_index_table(tab, out='int', bits=3)
    with pytest.raises(TypeError):
        vm.lookup(c, table)
    res = vm.lookup(ctx.load_encrypted_index(c.dumps()).decompress(ctx.thread), table)
    assert numpy.array_equal(ctx.decrypt_int(sk, res, 3), tab[values])


def test_compressed_multi_bit_cloud_key():
    import nufhe_b200 as nufhe
    ctx = nufhe.Context(rng=nufhe.DeterministicRNG(7))
    sk = ctx.make_secret_key()
    cck, ik = ctx.make_cloud_key(sk, compressed=True, multi_bit=2, index_key=True)
    vm = ctx.make_virtual_machine(cck.decompress(ctx.thread))
    rng = numpy.random.RandomState(9)
    values = rng.randint(0, 256, size=4096)
    tab = rng.randint(0, 2, size=256)
    res = vm.lookup(ctx.encrypt_index(ik, values, 8), vm.make_index_table(tab, out='bool'))
    assert numpy.array_equal(ctx.decrypt(sk, res), tab[values].astype(bool))


@pytest.mark.parametrize('m, W', [(10, 16), (16, 16), (20, 4)])
def test_output_noise(api, idx16, m, W):
    """4096 queries into a W-column table (65 536 outputs at m = 10 and 16, 16 384 at m = 20), before the key switch:
    the variance of the phase error lies within 0.5 to 2 times the estimate index_lookup.extracted_variance (m x
    1.84e-8), the mean error is below a tenth of a standard deviation (truncated digits shifted it coherently, by about
    -2.6e-4 at m = 16), and no error exceeds 7 sigma"""
    from nufhe_b200 import index_lookup as IL
    nufhe, ctx, sk, ik, vm = api
    if m == 16:
        values, e = idx16
    else:
        values = numpy.random.RandomState(m).randint(0, 1 << m, size=4096)
        e = ctx.encrypt_index(ik, values, m)
    tab = numpy.random.RandomState(18).randint(0, 4, size=(W, 1 << m))
    table = vm.make_index_table(tab, out='int', bits=2)
    a, b = IL.lookup_extracted(ctx.thread, e, table)
    key = ik.key.reshape(-1).to(a.device)
    phase = ctx.thread.lwe_dot(a.reshape(-1, N), key, add1=b.reshape(-1), sign=-1).cpu().numpy().reshape(W, -1)
    want = (tab[:, values].astype(numpy.int64) << 29)
    err = ((phase.astype(numpy.int64) - want + 2**31) % 2**32 - 2**31) / 2**32
    var = float((err**2).mean())
    est = IL.extracted_variance(nufhe.NuFHEParameters(), m)
    print('m = %d: variance %.3g, estimate %.3g (ratio %.2f), max |err| %.3g, mean %.3g'
          % (m, var, est, var / est, abs(err).max(), err.mean()))
    assert 0.5 * est <= var <= 2 * est
    assert abs(err.mean()) < 0.1 * est**0.5
    assert abs(err).max() < 7 * est**0.5
