"""Multi-bit bootstrap keys on the CPU (DESIGN.md section 14): the C oracle's exact multi-bit rotation and the float
reference rotation (tests/multibit_ref.py) against each other, against the oracle's standard bootstrap and against the
noiseless-key identity, the kernel's pass-3 model run by the host emulator against both bit for bit, the exactness bound at worst-case inputs, key generation on the oracle-backed engine double, and the
noise rules and argument checks of the Python layer."""
import ctypes
import hashlib
import os

import numpy
import pytest

import gen_inputs as G
import multibit_ref as M
from fake_engine import FakeEngine
from oracle import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 1024


@pytest.fixture(scope='module')
def emul():
    return ctypes.CDLL(os.path.join(ROOT, 'nufhe_b200', 'csrc', 'libnb_host_emul.so'))


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _random_ct(rng, B, n):
    a = rng.randint(-2**31, 2**31, size=(B, n), dtype=numpy.int64).astype(numpy.int32)
    b = rng.randint(-2**31, 2**31, size=B, dtype=numpy.int64).astype(numpy.int32)
    return a, b


# ---- the reference ---------------------------------------------------------------------------------------------------

def test_reference_standard_rotation_matches_the_oracle():
    """the reference's machinery, run as the standard rotation, gives the oracle's bootstrap bit for bit"""
    keys = O.OracleKeys(31, n=40)
    raw, ref = M.standard_key(keys, 32)
    rng = numpy.random.RandomState(1)
    a, b = _random_ct(rng, 3, keys.n)
    want = O.bootstrap(a, b, ref, None, O.MU)
    got = M.bootstrap_extract((a, b), None, 0, 1, 0, O.MU, raw, rotate=M.blind_rotate_std)
    assert numpy.array_equal(got[0], want[0]) and numpy.array_equal(got[1], want[1])


EDGE_ROT = [0, 1, N - 1, N, N + 1, 2 * N - 1]


def test_oracle_rotation_matches_reference_at_random_rotations():
    """the exact oracle's multi-bit rotation equals the float reference bit for bit: noisy key, random accumulators and
    rotations, n = 26"""
    keys = O.OracleKeys(37, n=26, make_bk=False)
    raw, ref = M.multibit_key(keys, 38)
    rng = numpy.random.RandomState(6)
    B = 8
    acc = rng.randint(-2**31, 2**31, size=(B, 2, N), dtype=numpy.int64).astype(numpy.int32)
    bara = rng.randint(0, 2 * N, size=(B, keys.n)).astype(numpy.int32)
    got = M.blind_rotate_oracle(acc, bara, ref)
    assert numpy.array_equal(got, M.blind_rotate_mb(acc, bara, raw))
    assert not numpy.array_equal(got, acc)


def test_oracle_rotation_matches_reference_at_every_edge_pair():
    """every ordered pair of the rotation edges 0, 1, N - 1, N, N + 1, 2N - 1 as some group's (abar_2g, abar_2g+1),
    including the pairs whose sum wraps past 2N: the oracle equals the float reference bit for bit"""
    keys = O.OracleKeys(39, n=36, make_bk=False)
    raw, ref = M.multibit_key(keys, 40)
    pairs = numpy.array([(x, y) for x in EDGE_ROT for y in EDGE_ROT], numpy.int32)      # 36 pairs
    rng = numpy.random.RandomState(7)
    B = 2
    acc = rng.randint(-2**31, 2**31, size=(B, 2, N), dtype=numpy.int64).astype(numpy.int32)
    bara = pairs.reshape(B, keys.n)
    assert (pairs.sum(1) >= 2 * N).any()
    assert numpy.array_equal(M.blind_rotate_oracle(acc, bara, ref), M.blind_rotate_mb(acc, bara, raw))


def test_oracle_rotation_refuses_bad_arguments():
    keys = O.OracleKeys(41, n=4, make_bk=False)
    ref = M.multibit_key(keys, 42)[1]
    acc = numpy.zeros((1, 2, N), numpy.int32)
    with pytest.raises(AssertionError):
        O.blind_rotate_mb(acc, ref, numpy.zeros((1, 3), numpy.int32))            # odd n
    with pytest.raises(AssertionError):
        O.blind_rotate_mb(acc, ref, numpy.zeros((1, 6), numpy.int32))            # fewer than n / 2 groups
    with pytest.raises(AssertionError):
        O.blind_rotate_mb(acc, ref, numpy.full((1, 4), 2 * N, numpy.int32))      # rotation outside [0, 2N)


@pytest.mark.parametrize('rotate', [M.blind_rotate_std, M.blind_rotate_mb, M.blind_rotate_oracle])
def test_noiseless_keys_rotate_exactly(rotate):
    """noiseless keys, test vectors of multiples of 2^12: every rotation gives exactly X^(sum abar_i s_i) tv"""
    keys = O.OracleKeys(33, n=64, make_bk=False)
    raw, ref = (M.standard_key if rotate is M.blind_rotate_std else M.multibit_key)(keys, 0, noiseless=True)
    raw = ref if rotate is M.blind_rotate_oracle else raw
    rng = numpy.random.RandomState(2)
    B = 6
    bara = rng.randint(0, 2 * N, size=(B, keys.n))
    bara[0] = 0
    bara[1] = N
    bara[2, ::3] = 2 * N - 1
    acc = numpy.zeros((B, 2, N), numpy.int32)
    acc[:, 1] = (rng.randint(0, 2**20, size=(B, N)) << 12).astype(numpy.uint32).view(numpy.int32)
    got = rotate(acc, bara, raw)
    e = (bara * keys.lwe_key).sum(-1)
    assert (got[:, 0] == 0).all()
    assert numpy.array_equal(got[:, 1], M.exact_rotation(acc[:, 1], e))


# ---- the kernel's pass 3 on the host ---------------------------------------------------------------------------------

def _group(emul, acc, rows_ref, rot):
    out = numpy.ascontiguousarray(acc.copy())
    assert emul.emul_fft_group_mb(_p(out), _p(numpy.ascontiguousarray(rows_ref)), _p(numpy.ascontiguousarray(rot, numpy.int32)),
                                  ctypes.c_int(acc.shape[0])) == 0
    return out


@pytest.mark.parametrize('case', ['random', 'worst'])
def test_emulated_group_matches_reference(emul, case):
    """one group of the kernel's multi-bit step (fwd1, fwd2, the 3-row pass 3, inv2, inv1; host emulator) against the
    float reference and the exact oracle, both ciphertext slots, for a noisy key and for keys at the extremes of the
    32-bit range with digits at -512 / 511"""
    rng = numpy.random.RandomState(3 if case == 'random' else 4)
    keys = O.OracleKeys(35, n=2, make_bk=False)
    if case == 'random':
        raw = M.multibit_key(keys, 36)[0]
        acc = rng.randint(-2**31, 2**31, size=(2, 2, N), dtype=numpy.int64).astype(numpy.int32)
        rots = [rng.randint(0, 2 * N, size=(2, 2)) for _ in range(4)] + [numpy.array([[0, N], [2 * N - 1, 1]])]
    else:
        raw = numpy.empty((3, 2, 2, 2, N), numpy.int32)
        pats = [numpy.full(N, -2**31), numpy.full(N, 2**31 - 1), numpy.where(numpy.arange(N) % 2, -2**31, 2**31 - 1),
                numpy.full(N, -2**31 + 2**15)]
        for i, idx in enumerate(numpy.ndindex(3, 2, 2, 2)):
            raw[idx] = pats[i % len(pats)]
        # accumulators whose digits are all -512 (t = acc + 2^31 + 2^21 = 0) or all 511 (t = 0xfffff000), and
        # alternating
        lo = numpy.int64(-(2**31 + 2**21)) & 0xffffffff
        hi = (numpy.int64(0xfffff000) - (2**31 + 2**21)) & 0xffffffff
        acc = numpy.empty((2, 2, N), numpy.int64)
        acc[0, 0], acc[0, 1] = lo, hi
        acc[1] = numpy.where(numpy.arange(N) % 2, lo, hi)
        acc = acc.astype(numpy.uint32).view(numpy.int32)
        rots = [numpy.array([[1, 1], [N - 1, N + 1]]), numpy.array([[N, N], [0, 2 * N - 1]])]
    ref = O.bk_transform(raw)
    for rot in rots:
        got = _group(emul, acc, ref, rot)
        want = M.blind_rotate_mb(acc, rot, raw)
        assert numpy.array_equal(got, want)
        assert numpy.array_equal(got, M.blind_rotate_oracle(acc, rot, ref))


def _negacyclic(a, b):
    """exact a * b mod X^N + 1 for int64 polynomials whose products and sums stay below 2^63"""
    k, i = numpy.meshgrid(numpy.arange(N), numpy.arange(N), indexing='ij')
    m = numpy.where(k >= i, b[(k - i) % N], -b[(k - i) % N])
    return m @ a


def _times_xk_minus_1(p, k):
    """(X^k - 1) p, exactly"""
    src = (numpy.arange(N) - k) % (2 * N)
    r = numpy.where(src >= N, -p[src % N], p[src % N])
    return r - p


def _halves(k):
    lo = ((k + 32768) & 65535) - 32768
    return lo, (k - lo) >> 16


@pytest.mark.parametrize('case', range(6))
def test_exactness_bound_at_worst_case(emul, case):
    """The unrounded multi-bit chain of the kernel (host emulator: fwd1, fwd2, the 3-row pass 3, inv2, inv1) against
    the exact sum_p (X^k_p - 1) sum_d dig_d key_{p,d},h at worst-case inputs -- digits all -512 / 511 or alternating,
    keys at -2^31, 2^31 - 1, alternating and wrap-aligned, rotations whose factors reach -2 -- stays within the bound
    of DESIGN.md section 14 (0.12), far from 1/2"""
    rng = numpy.random.RandomState(100 + case)
    idx = numpy.arange(N)
    digs = [numpy.full(N, -512), numpy.full(N, 511), numpy.where(idx % 2, -512, 511), numpy.where(idx < N // 2, 511, -512)]
    keys = [numpy.full(N, -2**31), numpy.full(N, 2**31 - 1), numpy.where(idx % 2, -2**31, 2**31 - 1),
            numpy.where(idx < N // 2, 2**31 - 1, -2**31), numpy.full(N, -2**31 + 2**15), numpy.full(N, 2**15 - 1)]
    dig = numpy.stack([digs[(case + d) % 4] if case < 4 else rng.choice([-512, 511], N) for d in range(4)]).astype(numpy.int64)
    key = numpy.stack([numpy.stack([keys[(case + p + 2 * d) % len(keys)] if case < 5 else rng.choice([-2**31, 2**31 - 1], N)
                                    for d in range(4)]) for p in range(3)]).astype(numpy.int64)
    rot = [(N, 0), (N // 2, N // 2), (N, N), (1, N - 1), (2 * N - 1, N + 1), (N, 2 * N - 1)][case]
    out = numpy.empty((2, N), numpy.float64)
    emul.emul_fft_product_mb(_p(numpy.ascontiguousarray(dig, numpy.float64)), _p(numpy.ascontiguousarray(key)),
                             _p(numpy.array(rot, numpy.int32)), _p(out))
    ks = (rot[0], rot[1], (rot[0] + rot[1]) % (2 * N))
    worst = 0.0
    for h in range(2):
        exact = sum(_times_xk_minus_1(sum(_negacyclic(dig[d], _halves(key[p, d])[h]) for d in range(4)), ks[p])
                    for p in range(3))
        assert numpy.abs(exact).max() < 6 * 2**36
        worst = max(worst, float(numpy.abs(out[h] - exact).max()))
    print('case %d: largest distance from the exact integer %.3g' % (case, worst))
    assert worst < 0.12


# ---- keys on the engine double ---------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def nufhe():
    import nufhe_b200
    return nufhe_b200


def _sha(t, unsigned=False):
    a = t.cpu().numpy()
    return hashlib.sha256(numpy.ascontiguousarray(a.view(numpy.uint64) if unsigned else a).tobytes()).hexdigest()


class _SeededFakeEngine(FakeEngine):
    """the engine double with Engine.seeded_uniform from the NumPy keystream (compressed keys)"""

    def seeded_uniform(self, seed, nonce, shape, first=0):
        import torch
        from chacha_ref import seeded_uniform
        return torch.from_numpy(numpy.ascontiguousarray(seeded_uniform(seed, nonce, shape, first)))


def _ctx(nufhe, seed):
    return nufhe.Context(rng=nufhe.DeterministicRNG(seed), thread=_SeededFakeEngine())


def test_multi_bit_1_keeps_the_golden_keys(nufhe, golden):
    g = golden('gate')
    ctx = _ctx(nufhe, G.GATE_SEED)
    sk = ctx.make_secret_key()
    ck = ctx.make_cloud_key(sk, multi_bit=1)
    assert type(ck.bootstrap_key) is nufhe.bootstrap.BootstrapKey
    assert _sha(ck.bootstrap_key.tgsw.samples.a.coeffs, True) == str(g['bk_sha'])
    assert _sha(ck.keyswitch_key.lwe.a) == str(g['ks_a_sha']) and _sha(ck.keyswitch_key.lwe.b) == str(g['ks_b_sha'])


@pytest.fixture(scope='module')
def mb(nufhe):
    ctx = _ctx(nufhe, 77)
    sk = ctx.make_secret_key()
    ck = ctx.make_cloud_key(sk, multi_bit=2)
    return ctx, sk, ck


def test_draw_order_and_rows_decrypt_to_their_indicators(nufhe, mb):
    """the multi-bit rows take the bootstrap key's place in the draws: replaying them (TGSW key, then 750 TGSW
    encryptions of the indicators in row order, then the key-switch key) gives the same cloud key, and every row's
    body level j has phase [s_2g = b0 and s_2g+1 = b1] 2^(22 - 10 j) at coefficient 0 plus small noise"""
    from nufhe_b200.tgsw import TGswKey, TGswSampleArray, tgsw_encrypt_int, tgsw_transform_samples
    from nufhe_b200.bootstrap import MultiBitTGswSampleArray, multi_bit_messages
    from nufhe_b200.lwe import LweKeyswitchKey
    ctx, sk, ck = mb
    assert isinstance(ck.bootstrap_key, nufhe.MultiBitBootstrapKey) and ck.bootstrap_key.tgsw.shape == (750,)
    ctx2 = _ctx(nufhe, 77)
    sk2 = ctx2.make_secret_key()
    thr, rng, params = ctx2.thread, ctx2.rng, sk2.params
    tgsw_key = TGswKey.from_rng(thr, params.tgsw_params, rng)
    msgs = multi_bit_messages(sk2.lwe_key.key)
    assert numpy.array_equal(msgs.numpy(), M.indicators(sk2.lwe_key.key.numpy()))
    rows = TGswSampleArray.empty(thr, params.tgsw_params, (750,))
    tgsw_encrypt_int(thr, rng, rows, msgs, params.tgsw_params.tlwe_params.min_noise, tgsw_key)
    tr = MultiBitTGswSampleArray.empty(thr, params.tgsw_params, (750,))
    tgsw_transform_samples(thr, tr, rows)
    ks = LweKeyswitchKey.from_tgsw_key(thr, rng, params.ks_decomp_length, params.ks_log2_base, sk2.lwe_key, tgsw_key)
    assert tr == ck.bootstrap_key.tgsw and ks == ck.keyswitch_key
    c = rows.samples.a.coeffs.numpy()                                          # (750, mi, j, mo, N)
    S = tgsw_key.tlwe_key.key.coeffs.numpy()[0]
    mask = numpy.ascontiguousarray(c[:, 1, :, 0])
    phase = (c[:, 1, :, 1].astype(numpy.int64) - O.poly_mul_i32(S, mask).astype(numpy.int64)) & 0xffffffff
    phase = numpy.where(phase >= 2**31, phase - 2**32, phase)
    expect = numpy.zeros_like(phase)
    expect[:, 0, 0] = msgs.numpy() * 2**22
    expect[:, 1, 0] = msgs.numpy() * 2**12
    assert numpy.abs(phase - expect).max() < 2**10


def test_pickles_round_trip(nufhe, mb):
    ctx, sk, ck = mb
    blob = ck.dumps()
    back = ctx.load_cloud_key(blob)
    assert back == ck and isinstance(back.bootstrap_key, nufhe.MultiBitBootstrapKey)
    assert b'nufhe_b200.MultiBitBootstrapKey/1' in blob
    # a standard key's pickle carries no tag and loads as before
    std = _ctx(nufhe, 78)
    ck2 = std.make_cloud_key(std.make_secret_key())
    blob2 = ck2.dumps()
    assert b'MultiBitBootstrapKey' not in blob2 and std.load_cloud_key(blob2) == ck2


def test_compressed_multi_bit_key(nufhe):
    """compressed: 750 bodies, masks from the seed; decompress() gives a MultiBitBootstrapKey, through a pickle as well;
    compressed multi_bit=1 keeps today's draws"""
    ctx = _ctx(nufhe, 79)
    sk = ctx.make_secret_key()
    cck = ctx.make_cloud_key(sk, compressed=True, multi_bit=2)
    assert tuple(cck.bk_body.shape) == (750, 2, 2, 1024)
    # the mask stream of the bootstrap key continues over all 750 rows (DESIGN.md section 10)
    from chacha_ref import seeded_uniform
    from nufhe_b200 import compressed as C
    masks = seeded_uniform(cck.seed, C.NONCE_BOOTSTRAP_KEY, (750, 2, 2, 1, 1024))
    first = seeded_uniform(cck.seed, C.NONCE_BOOTSTRAP_KEY, (500, 2, 2, 1, 1024))
    assert numpy.array_equal(masks[:500], first)
    back = ctx.load_compressed_cloud_key(cck.dumps())
    assert back == cck
    ck = back.decompress(ctx.thread)
    assert isinstance(ck.bootstrap_key, nufhe.MultiBitBootstrapKey) and ck.bootstrap_key.tgsw.shape == (750,)
    a, b = _ctx(nufhe, 80), _ctx(nufhe, 80)
    ska, skb = a.make_secret_key(), b.make_secret_key()
    assert a.make_cloud_key(ska, compressed=True) == b.make_cloud_key(skb, compressed=True, multi_bit=1)


def test_argument_checks(nufhe):
    import types
    from nufhe_b200.bootstrap import check_multi_bit
    ctx = _ctx(nufhe, 81)
    sk = ctx.make_secret_key()
    for bad in (0, 3, -1):
        with pytest.raises(ValueError):
            ctx.make_cloud_key(sk, multi_bit=bad)
    for bad in ('2', 2.0, True, None):
        with pytest.raises(TypeError):
            ctx.make_cloud_key(sk, multi_bit=bad)
    k2 = ctx.make_secret_key(tlwe_mask_size=2)
    for compressed in (False, True):
        with pytest.raises(ValueError):
            ctx.make_cloud_key(k2, compressed=compressed, multi_bit=2)
    params = nufhe.NuFHEParameters()
    odd = types.SimpleNamespace(tgsw_params=params.tgsw_params, in_out_params=types.SimpleNamespace(size=501))
    with pytest.raises(ValueError, match='even'):
        check_multi_bit(odd, 2)
    check_multi_bit(odd, 1)


def test_single_kernel_false_is_refused(nufhe, mb):
    ctx, sk, ck = mb
    with pytest.raises(ValueError, match='fused'):
        ctx.make_virtual_machine(ck, perf_params=nufhe.PerformanceParameters(ck.params, single_kernel_bootstrap=False))


# ---- noise rules -----------------------------------------------------------------------------------------------------

def _allowed(params, multi_bit):
    from nufhe_b200 import lut
    return {(P, L, sh) for P in (1, 2, 3) for L in (0, 1, 2) for sh in [None] + list(range(P))
            if 2.0**-(P + 2) / lut.lut_sigma(params, L, sh, multi_bit) >= lut.MARGIN_SIGMAS}


def test_noise_rules(nufhe):
    from nufhe_b200 import lut, tree_lut
    params = nufhe.NuFHEParameters()
    assert _allowed(params, 1) == lut.ALLOWED
    assert _allowed(params, 2) == lut.ALLOWED_MULTI_BIT
    # the key term: (n / 2) groups x 3 rows x 2 (the factor X^k - 1) external products against n
    ks = 1024 * 8 * 3 / 4 * params.in_out_params.min_noise**2
    br1, br2 = lut.bootstrap_variance(params, 1) - ks, lut.bootstrap_variance(params, 2) - ks
    assert abs(br2 / br1 - 3) < 1e-9 and 2.7e-5 < br2 < 2.9e-5
    # a gate whose inputs are two gate outputs keeps about 15 sigma
    assert 15 < 0.125 / (2 * lut.bootstrap_variance(params, 2))**0.5 < 16.5
    assert tree_lut.max_digits(params, 2, 1) == 4 and tree_lut.max_digits(params, 2, 2) == 2
    lut.check_noise(params, 2, 1, 0)
    with pytest.raises(ValueError):
        lut.check_noise(params, 2, 1, 0, multi_bit=2)
    with pytest.raises(ValueError):
        tree_lut.TreeLookupTable(FakeEngine(), params, numpy.zeros((4, 4, 4), int), 2, 3, multi_bit=2)
