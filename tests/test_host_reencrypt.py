"""Re-encryption on the CPU (DESIGN.md section 22): the NumPy reference (reencrypt_ref.py) against a trivially encrypted
key, the tree-key composition and worst-case digits; the index functions of csrc/reencrypt_layout.cuh through the host
emulator; make_reencryption_key (draw order, phase, pickles, argument errors); vm.reencrypt and mk.reencrypt on the
engine double (tests/reencrypt_fake.py): decryption under the recipient's key, gates on the results, multi-key identity
on resident and compressed keys, variance bookkeeping, the input-variance limit and the margin table."""
import copy
import ctypes
import io
import os

import numpy
import pytest

import nufhe_b200
from nufhe_b200 import reencrypt, lut, index_lookup, compact
from nufhe_b200.compressed import draw_seed
from nufhe_b200.lut import encode_int
from nufhe_b200.random_numbers import DeterministicRNG
from chacha_ref import seeded_uniform
from fake_engine import _np, _t
from oracle import oracle as O
from pack_ref import digits, u32, i32
from reencrypt_fake import ReencryptFakeEngine
import compact_ref
import reencrypt_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 1024
n = 500
SIGMA = 9e-9 * (2 / numpy.pi)**0.5
ALL_MINUS = 0x7f7f8000                       # a word whose two digits are -128
ALL_PLUS = 0x7f7e8000                        # a word whose two digits are 127


@pytest.fixture(scope='module')
def emul():
    path = os.path.join(ROOT, 'nufhe_b200', 'csrc', 'libnb_host_emul.so')
    if not os.path.exists(path):
        import __graft_entry__ as g
        g.build()
    lib = ctypes.CDLL(path)
    lib.emul_reenc_slot.argtypes = [ctypes.c_uint32, ctypes.c_int]
    lib.emul_reenc_slot.restype = ctypes.c_uint32
    lib.emul_reenc_coeff.argtypes = [ctypes.c_uint32]
    lib.emul_reenc_coeff.restype = ctypes.c_uint32
    lib.emul_reenc_negated.argtypes = [ctypes.c_uint32]
    lib.emul_reenc_negated.restype = ctypes.c_int
    lib.emul_reenc_digits.argtypes = [ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p]
    lib.emul_reenc_digits.restype = None
    lib.emul_reenc_mask.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    lib.emul_reenc_mask.restype = None
    return lib


def _emul_digits(emul, a):
    a = numpy.ascontiguousarray(a, numpy.int32)
    out = numpy.empty(N, numpy.int32)
    emul.emul_reenc_digits(a.ctypes.data, a.size, out.ctypes.data)
    return out


def _emul_mask(emul, prod):
    p = numpy.ascontiguousarray(u32(prod).astype(numpy.uint32))
    out = numpy.empty(N, numpy.int32)
    emul.emul_reenc_mask(p.ctypes.data, out.ctypes.data)
    return out


def _random_key(seed):
    rng = numpy.random.RandomState(seed)
    return (rng.randint(-2**31, 2**31, size=N, dtype=numpy.int64).astype(numpy.int32),
            rng.randint(-2**31, 2**31, size=N, dtype=numpy.int64).astype(numpy.int32))


def _random_samples(seed, R):
    rng = numpy.random.RandomState(seed)
    a = rng.randint(-2**31, 2**31, size=(R, n), dtype=numpy.int64).astype(numpy.int32)
    b = rng.randint(-2**31, 2**31, size=R, dtype=numpy.int64).astype(numpy.int32)
    return a, b


# ---------------------------------------------------------------- the reference and the header

def test_worst_case_words():
    assert (digits(numpy.array([ALL_MINUS], numpy.int64)) == -128).all()
    assert (digits(numpy.array([ALL_PLUS], numpy.int64)) == 127).all()


def test_reference_with_trivial_key():
    """Zero mask and no noise: the result is (0, b - sum_i s_A[i] round_16(a_i)) exactly."""
    rng = numpy.random.RandomState(1)
    s = rng.randint(0, 2, size=n)
    body = numpy.zeros(N, numpy.int64)
    body[0:2 * n:2] = s * 2**24
    body[1:2 * n:2] = s * 2**16
    a, b = _random_samples(2, 16)
    a[0] = ALL_MINUS
    a[1] = ALL_PLUS
    out_a, out_b = reencrypt_ref.reencrypt(a, b, numpy.zeros(N, numpy.int32), i32(body))
    assert (out_a == 0).all()
    rounded = u32(a.astype(numpy.int64) + 2**15) >> 16 << 16
    assert (out_b == i32(b.astype(numpy.int64) - rounded @ s)).all()


@pytest.mark.parametrize('case', ['random', 'minus', 'plus'])
def test_reference_against_tree_chain(case):
    """Random int32 keys: the literal definition equals the tree-key composition of the rotations X^(-p) C, bit for bit,
    on random masks and on masks whose digits are all -128 or all 127."""
    mask, body = _random_key(3)
    a, b = _random_samples(4, 8)
    if case == 'minus':
        a[:] = ALL_MINUS
    elif case == 'plus':
        a[:] = ALL_PLUS
    got = reencrypt_ref.reencrypt(a, b, mask, body)
    want = reencrypt_ref.tree_chain(a, b, mask, body)
    assert (got[0] == want[0]).all() and (got[1] == want[1]).all()


def test_header_index_functions(emul):
    for p in range(N):
        assert emul.emul_reenc_coeff(p) == (N - p) % N
        assert emul.emul_reenc_coeff(emul.emul_reenc_coeff(p)) == p
        assert emul.emul_reenc_negated(p) == (p == 0)
    for i in (0, 1, 249, n - 1):
        for j in (0, 1):
            assert emul.emul_reenc_slot(i, j) == 2 * i + j
    # -D of one mask: coefficient 0 holds -d_0, coefficient N - p holds d_p, zero where no digit lands
    a, _ = _random_samples(5, 1)
    d = digits(a[0]).reshape(-1)
    want = numpy.zeros(N, numpy.int64)
    want[0] = -d[0]
    for p in range(1, 2 * n):
        want[N - p] = d[p]
    assert (_emul_digits(emul, a[0]) == want).all()
    assert (_emul_digits(emul, a[0, :3])[1:N - 5] == 0).all()          # n = 3: digits 0..5 only
    # the output mask is the negated slot-0 extraction of the product by D, i.e. the slot-0 extraction by -D
    prod = numpy.random.RandomState(6).randint(-2**31, 2**31, size=N, dtype=numpy.int64)
    got = _emul_mask(emul, prod)
    assert got[0] == i32(prod[0]) and (got[1:] == i32(-prod[:0:-1])).all()
    assert (got == i32(reencrypt_ref.extraction_matrix(prod)[0])).all()


@pytest.mark.parametrize('case', ['random', 'minus', 'plus'])
def test_header_composition(emul, case):
    """The kernel's route: -D from the header, an exact negacyclic product with the mask, the header's extraction and
    the body dot product, equals the reference."""
    mask, body = _random_key(7)
    a, b = _random_samples(8, 4)
    if case != 'random':
        a[:] = ALL_MINUS if case == 'minus' else ALL_PLUS
    M = compact_ref.negacyclic_matrix(u32(mask))
    want_a, want_b = reencrypt_ref.reencrypt(a, b, mask, body)
    for r in range(a.shape[0]):
        D = _emul_digits(emul, a[r]).astype(numpy.int64)
        prod = u32(D @ M)                                 # |sum| < 1000 * 128 * 2^32 < 2^63
        assert (_emul_mask(emul, prod) == want_a[r]).all()
        d = numpy.where(numpy.arange(N) == 0, -D, D)[(N - numpy.arange(N)) % N]   # d_p at p
        assert i32(b[r].astype(numpy.int64) - d @ body.astype(numpy.int64)) == want_b[r]


# ---------------------------------------------------------------- the key

def _client(thr, seed, compressed=False):
    ctx = nufhe_b200.Context(rng=DeterministicRNG(seed), thread=thr)
    sk = ctx.make_secret_key()
    ck, cpk = ctx.make_cloud_key(sk, compressed=compressed, compact_public_key=True)
    replay = DeterministicRNG(seed)
    replay.uniform_bool((n,))
    S = replay.uniform_bool((1, N))[0]                  # the bootstrap key's GLWE key, drawn first by make_cloud_key
    vck = ck.decompress(thr) if compressed else ck
    return dict(ctx=ctx, sk=sk, ck=ck, cpk=cpk, S=S, vm=ctx.make_virtual_machine(vck))


@pytest.fixture(scope='module')
def env():
    thr = ReencryptFakeEngine()
    sender = _client(thr, 7001)
    recipients = [_client(thr, 7100 + i, compressed=True) for i in range(3)]
    return dict(thr=thr, A=sender, Bs=recipients)


def _key_polys(cpk):
    return numpy.concatenate([seeded_uniform(cpk.seed, compact.NONCE_COMPACT_KEY, (1, N)), _np(cpk.b)[None]])


def test_key_draw_order_and_phase(env):
    A, B = env['A'], env['Bs'][0]
    ctx = A['ctx']
    replay = copy.deepcopy(ctx.rng)
    rekey = ctx.make_reencryption_key(A['sk'], B['cpk'])
    assert isinstance(rekey, nufhe_b200.NuFHEReencryptionKey) and rekey.n == n
    r_seed = draw_seed(replay)
    e1 = O.double_to_t32(replay.gauss((1, 1, N), SIGMA)).astype(numpy.int64)
    e2 = O.double_to_t32(replay.gauss((1, N), SIGMA)).astype(numpy.int64)
    words = seeded_uniform(r_seed, compact.NONCE_COMPACT_RANDOMNESS, (1, N // 32))
    C = compact_ref.products(_key_polys(B['cpk']), compact_ref.r_bits(words))[0]
    s = _np(A['sk'].lwe_key.key).astype(numpy.int64)
    mus = numpy.zeros(N, numpy.int64)
    mus[0:2 * n:2], mus[1:2 * n:2] = s * 2**24, s * 2**16
    want = C.copy()
    want[0] += e1[0, 0]
    want[1] += e2[0] + mus
    assert (_np(rekey.sample) == i32(want)).all()                   # unrounded: every bit of the sums is kept
    # decrypted under S_B: s_A[i] g_j at slot 2 i + j within the fresh noise, 0 from slot 2 n on
    sample = _np(rekey.sample).astype(numpy.int64)
    ph = i32(sample[1] - sample[0] @ compact_ref.negacyclic_matrix(B['S'])).astype(numpy.int64)
    err = i32(ph - mus).astype(numpy.float64) / 2**32
    assert numpy.abs(err).max() < 8 * reencrypt.noise_terms(B['ck'].params)[0]**0.5
    assert numpy.abs(err[2 * n:]).max() < 8 * reencrypt.noise_terms(B['ck'].params)[0]**0.5


def test_key_pickles(env):
    A, B = env['A'], env['Bs'][1]
    ctx = A['ctx']
    rekey = ctx.make_reencryption_key(A['sk'], B['cpk'])
    s = rekey.dumps()
    assert 8192 < len(s) < 9500
    assert ctx.load_reencryption_key(s) == rekey and ctx.load_reencryption_key(io.BytesIO(s)) == rekey
    for wrong in (B['cpk'].dumps(), A['sk'].dumps(), b'junk'):
        with pytest.raises(ValueError):
            ctx.load_reencryption_key(wrong)
    with pytest.raises(ValueError):
        ctx.load_reencryption_key(s[:-100])
    with pytest.raises(ValueError):
        ctx.load_compact_public_key(s)


def test_key_argument_errors(env):
    A, B = env['A'], env['Bs'][0]
    ctx = A['ctx']
    with pytest.raises(TypeError):
        ctx.make_reencryption_key(B['cpk'], B['cpk'])
    with pytest.raises(TypeError):
        ctx.make_reencryption_key(A['sk'], A['sk'])
    with pytest.raises(TypeError):
        ctx.make_reencryption_key(A['sk'], B['ck'])
    other = ctx.make_secret_key(tlwe_mask_size=2)
    with pytest.raises(ValueError):
        ctx.make_reencryption_key(other, B['cpk'])


# ---------------------------------------------------------------- the server

def _same(x, y):
    return (tuple(x.shape) == tuple(y.shape) and (_np(x.a) == _np(y.a)).all() and (_np(x.b) == _np(y.b)).all()
            and (_np(x.current_variances) == _np(y.current_variances)).all())


def test_vm_reencrypt_bits_ints_and_gate(env):
    A, B = env['A'], env['Bs'][0]
    ctx, vm = A['ctx'], B['vm']
    rekey = ctx.make_reencryption_key(A['sk'], B['cpk'])
    bits = numpy.array([[True, False, True], [False, True, True]])
    ct = ctx.encrypt(A['sk'], bits)
    out = vm.reencrypt(rekey, ct)
    assert isinstance(out, nufhe_b200.LweSampleArray) and out.shape == bits.shape
    assert (B['ctx'].decrypt(B['sk'], out) == bits).all()
    # the result against the reference and the recipient's key switch, and its variances
    mask = _np(rekey.sample)[0]
    ra, rb = reencrypt_ref.reencrypt(_np(ct.a).reshape(-1, n), _np(ct.b), mask, _np(rekey.sample)[1])
    ks = tuple(_np(x) for x in B['vm'].cloud_key.keyswitch_key.device_arrays())
    ka, kb, kcv = compact_ref.keyswitch(ks, ra, rb)
    assert (_np(out.a).reshape(ka.shape) == ka).all() and (_np(out.b).reshape(-1) == kb).all()
    want_cv = _np(ct.current_variances).reshape(-1) + kcv + reencrypt.reencrypt_variance(vm.params)
    assert numpy.allclose(_np(out.current_variances).reshape(-1), want_cv, rtol=1e-6)
    # a gate with the recipient's own bits
    mine = numpy.array([[True, True, False], [False, False, True]])
    nand = vm.gate_nand(out, B['ctx'].encrypt(B['sk'], mine))
    assert (B['ctx'].decrypt(B['sk'], nand) == ~(bits & mine)).all()
    # 2-bit integers
    values = numpy.array([0, 1, 2, 3, 3, 1])
    iv = vm.reencrypt(rekey, ctx.encrypt_int(A['sk'], values, 2))
    assert (B['ctx'].decrypt_int(B['sk'], iv, 2) == values).all()
    # into dest
    dest = vm.empty_ciphertext(bits.shape)
    assert vm.reencrypt(rekey, ct, dest=dest) is dest and _same(dest, out)


def test_vm_reencrypt_errors_and_variance_limit(env):
    A, B = env['A'], env['Bs'][0]
    ctx, vm = A['ctx'], B['vm']
    rekey = ctx.make_reencryption_key(A['sk'], B['cpk'])
    ct = ctx.encrypt(A['sk'], [True, False])
    with pytest.raises(TypeError):
        vm.reencrypt(B['cpk'], ct)
    with pytest.raises(TypeError):
        vm.reencrypt(rekey, B['ctx'].encrypt(B['cpk'], [True]))
    short = nufhe_b200.LweSampleArray(ct.params, ct.a[:, :400].contiguous(), ct.b, ct.current_variances)
    with pytest.raises(ValueError):
        vm.reencrypt(rekey, short)
    other = copy.copy(rekey)
    other.params = nufhe_b200.NuFHEParameters(tlwe_mask_size=2)
    with pytest.raises(ValueError):
        vm.reencrypt(other, ct)
    with pytest.raises(ValueError):
        vm.reencrypt(rekey, ct, dest=vm.empty_ciphertext((3,)))
    limit = reencrypt.MAX_INPUT_VARIANCE
    assert limit == reencrypt.max_input_variance(vm.params)
    ct.current_variances.fill_(limit * 0.999)
    vm.reencrypt(rekey, ct)
    ct.current_variances.fill_(limit * 1.001)
    with pytest.raises(ValueError):
        vm.reencrypt(rekey, ct)


def _mk_operands(env, R):
    A = env['A']
    ctx = A['ctx']
    rekeys, cts = [], []
    for t, B in enumerate(env['Bs']):
        rekeys.append(ctx.make_reencryption_key(A['sk'], B['cpk']))
        bits = numpy.random.RandomState(30 + t).randint(0, 2, size=(2 + 3 * t,)).astype(bool)
        cts.append(ctx.encrypt(A['sk'], bits))
    return rekeys + [None], cts + [None]


@pytest.mark.parametrize('R', [None, 2])
def test_mk_reencrypt_matches_per_tenant(env, R):
    """3 tenants plus an idle one, on resident keys and in rounds on compressed keys at R = 2."""
    A, Bs, thr = env['A'], env['Bs'], env['thr']
    ctx = A['ctx']
    rekeys, cts = _mk_operands(env, R)
    cks = [B['ck'] for B in Bs] + [Bs[0]['ck']]
    if R is None:
        mk = ctx.make_multi_key_machine([ck.decompress(thr) for ck in cks])
    else:
        mk = ctx.make_multi_key_machine(cks, resident_tenants=R)
    calls = thr.calls.get('reencrypt', 0)
    thr.reencrypt_segments = []
    got = mk.reencrypt(rekeys, cts)
    assert got[3] is None
    if R is None:
        assert thr.calls['reencrypt'] - calls == 1 and thr.reencrypt_segments == [[2, 5, 8]]
    for t, B in enumerate(Bs):
        want = B['vm'].reencrypt(rekeys[t], cts[t])
        assert _same(got[t], want), t
        assert (B['ctx'].decrypt(B['sk'], got[t]) == ctx.decrypt(A['sk'], cts[t])).all()
    with pytest.raises(ValueError):
        mk.reencrypt(rekeys[:2], cts)
    with pytest.raises(TypeError):
        mk.reencrypt([Bs[0]['cpk']] + rekeys[1:], cts)


# ---------------------------------------------------------------- noise

def test_noise_figures_and_margin_table():
    p = nufhe_b200.NuFHEParameters()
    fresh = ((2 * N) / 2 + 1) * SIGMA**2
    key_term = n * 2 * 5461.5 * fresh
    rounding = n / 2 * 2.0**-32 / 12
    assert reencrypt.DIGIT_SQUARE == 5461.5
    assert abs(key_term - 2.89e-7) < 0.01e-7 and abs(rounding - 4.9e-9) < 0.05e-9
    assert abs(reencrypt.reencrypt_variance(p) - (key_term + rounding)) < 1e-12 * key_term + 1e-20
    ks = index_lookup.keyswitch_variance(p)
    assert abs(ks - 3.64e-6) < 0.01e-6
    # rounding the key to 16 bits would have added 1000 x 5461.5 x 9.9e-9 = 0.054
    assert abs(2 * n * 5461.5 * (N / 2 + 1) * 2.0**-32 / 12 - 0.054) < 0.001
    total = lut.bootstrap_variance(p) + reencrypt.reencrypt_variance(p) + ks
    assert abs(total - 1.68e-5) < 0.01e-5 and total < 1.72e-5
    # the margin of a re-encrypted LUT output in every lut.ALLOWED configuration, re-derived
    table = reencrypt.margins(p)
    assert set(table) == set(lut.ALLOWED)
    for (P, L, sh), margin in table.items():
        weight = 1 if sh is None else 4**sh + 1
        sigma = (lut.lut_sigma(p, L, sh)**2 + weight * (reencrypt.reencrypt_variance(p) + ks))**0.5
        assert abs(margin - 2.0**-(P + 2) / sigma) < 1e-9 * margin
        assert margin >= 7.9
    assert abs(min(table.values()) - 7.97) < 0.01
    # the input limit: dozens of hops of re-encryption and key switch
    limit = reencrypt.MAX_INPUT_VARIANCE
    assert abs(limit - ((1 / 56)**2 - lut.lut_sigma(p, 0, 0)**2 - reencrypt.reencrypt_variance(p))) < 1e-15
    assert 60 < limit / (reencrypt.reencrypt_variance(p) + ks) < 80
