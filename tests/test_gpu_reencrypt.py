"""Re-encryption on the GPU (DESIGN.md section 22): nb_reencrypt bit-exact against the NumPy reference
(reencrypt_ref.py) at 1 to 4096 rows, with random and real keys, worst-case digits and several segments; against the
nb_tree_prepare -> nb_tree_keyswitch -> coefficient-0 chain; the C ABI's refusals; bits and 2-bit integers moved from one
client to another and used in gates and LUTs; the multi-key machine against per-tenant machines; and the measured noise
before and after the recipient's key switch."""
import ctypes

import numpy
import pytest
import torch

import compact_ref
import reencrypt_ref
from pack_ref import i32

pytestmark = pytest.mark.gpu
N = 1024
n = 500
ALL_MINUS, ALL_PLUS = 0x7f7f8000, 0x7f7e8000          # words whose two digits are -128, and 127


@pytest.fixture(scope='module')
def eng():
    from nufhe_b200.engine import Engine
    return Engine()


def _client(nufhe, ctx, multi_bit=1):
    sk = ctx.make_secret_key()
    ck, ik, cpk = ctx.make_cloud_key(sk, multi_bit=multi_bit, index_key=True, compact_public_key=True)
    return dict(sk=sk, ck=ck, S=ik.key.reshape(-1), cpk=cpk, vm=ctx.make_virtual_machine(ck))


@pytest.fixture(scope='module')
def api():
    import nufhe_b200
    ctx = nufhe_b200.Context(rng=nufhe_b200.DeterministicRNG(2210))
    A, B = _client(nufhe_b200, ctx), _client(nufhe_b200, ctx)
    return nufhe_b200, ctx, A, B


def _random_key(seed):
    rng = numpy.random.RandomState(seed)
    return tuple(rng.randint(-2**31, 2**31, size=N, dtype=numpy.int64).astype(numpy.int32) for _ in range(2))


def _samples(seed, R, case='random'):
    rng = numpy.random.RandomState(seed)
    a = rng.randint(-2**31, 2**31, size=(R, n), dtype=numpy.int64).astype(numpy.int32)
    b = rng.randint(-2**31, 2**31, size=R, dtype=numpy.int64).astype(numpy.int32)
    if case == 'minus':
        a[:] = ALL_MINUS
    elif case == 'plus':
        a[:] = ALL_PLUS
    return a, b


def _run(eng, a, b, keys, counts):
    specs = [eng.ntt_forward_i32(eng.to_device(m[None])) for m, _ in keys]
    bodies = [eng.to_device(x) for _, x in keys]
    out_a, out_b = eng.reencrypt(eng.to_device(a), eng.to_device(b), specs, bodies, counts)
    return out_a.cpu().numpy(), out_b.cpu().numpy()


@pytest.mark.parametrize('rows', [1, 2, 3, 257, 4096])
def test_kernel_random_keys(eng, rows):
    mask, body = _random_key(rows)
    a, b = _samples(rows + 1, rows)
    got = _run(eng, a, b, [(mask, body)], [rows])
    want = reencrypt_ref.reencrypt(a, b, mask, body)
    assert (got[0] == want[0]).all() and (got[1] == want[1]).all()


@pytest.mark.parametrize('case', ['minus', 'plus'])
def test_kernel_worst_case_digits(eng, case):
    mask, body = _random_key(5)
    a, b = _samples(6, 257, case)
    got = _run(eng, a, b, [(mask, body)], [257])
    want = reencrypt_ref.reencrypt(a, b, mask, body)
    assert (got[0] == want[0]).all() and (got[1] == want[1]).all()


def test_kernel_segments(eng):
    """Counts of 0 and counts that are not multiples of a CTA's 4 rows, each segment with its own key."""
    counts = [0, 5, 0, 3, 257, 1, 0, 4, 130]
    keys = [_random_key(100 + q) for q in range(len(counts))]
    a, b = _samples(7, sum(counts))
    got = _run(eng, a, b, keys, counts)
    lo = 0
    for (mask, body), c in zip(keys, counts):
        want = reencrypt_ref.reencrypt(a[lo:lo + c], b[lo:lo + c], mask, body)
        assert (got[0][lo:lo + c] == want[0]).all() and (got[1][lo:lo + c] == want[1]).all(), (lo, c)
        lo += c


def test_kernel_real_key_and_tree_chain(eng, api):
    """A real key at 4096 rows of real ciphertexts: the reference, and the tree-key chain on the GPU (nb_tree_prepare of
    the rotations X^(-p) C, nb_tree_keyswitch, coefficient 0), bit for bit."""
    nufhe, ctx, A, B = api
    rekey = ctx.make_reencryption_key(A['sk'], B['cpk'])
    bits = numpy.random.RandomState(8).randint(0, 2, size=4096).astype(bool)
    ct = ctx.encrypt(A['sk'], bits)
    a, b = ct.a.cpu().numpy(), ct.b.cpu().numpy()
    mask, body = rekey.sample.cpu().numpy()
    spec, bdy = rekey.spectra(eng)
    got = eng.reencrypt(ct.a, ct.b, [spec], [bdy], [4096])
    got = got[0].cpu().numpy(), got[1].cpu().numpy()
    want = reencrypt_ref.reencrypt(a, b, mask, body)
    assert (got[0] == want[0]).all() and (got[1] == want[1]).all()
    masks, bodies = reencrypt_ref.tree_key(mask, body, n)
    planes = eng.tree_prepare(eng.to_device(masks), eng.to_device(bodies))
    V = eng.tree_keyswitch(ct.a, planes, 1).cpu().numpy()
    chain = reencrypt_ref.from_tree_output(V, b)
    assert (got[0] == chain[0]).all() and (got[1] == chain[1]).all()


def test_capi_refusals(eng):
    lib, h = eng.lib, eng.handle
    a = torch.zeros((8, n), dtype=torch.int32, device=eng.device)
    b = torch.zeros(8, dtype=torch.int32, device=eng.device)
    spec = torch.zeros(N + 2, dtype=torch.int64, device=eng.device)
    body = torch.zeros(N + 1, dtype=torch.int32, device=eng.device)
    out_a = torch.zeros(8 * N + 4, dtype=torch.int32, device=eng.device)
    out_b = torch.zeros(8, dtype=torch.int32, device=eng.device)
    P = lambda t, off=0: ctypes.c_void_p(t.data_ptr() + off * t.element_size())
    arr = lambda ct, v: (ct * len(v))(*v)

    def call(a_=P(a), n_=n, k=1, specs=None, bodies=None, counts=(8,), oa=P(out_a), rows=8):
        specs = arr(ctypes.c_void_p, [spec.data_ptr()] * len(counts)) if specs is None else specs
        bodies = arr(ctypes.c_void_p, [body.data_ptr()] * len(counts)) if bodies is None else bodies
        rc = lib.nb_reencrypt(h, a_, P(b), n_, k, specs, bodies, arr(ctypes.c_size_t, list(counts)), len(counts), oa,
                              P(out_b), rows)
        return rc, lib.nb_last_error(h).decode()

    assert call()[0] == 0
    rc, msg = call(a_=None)
    assert rc == -1 and 'null argument' in msg
    rc, msg = call(specs=arr(ctypes.c_void_p, [None]))
    assert rc == -1 and 'null key of tenant 0' in msg
    rc, msg = call(oa=P(out_a, 1))
    assert rc == -1 and 'aligned' in msg
    rc, msg = call(specs=arr(ctypes.c_void_p, [spec.data_ptr() + 8]))
    assert rc == -1 and 'aligned' in msg
    rc, msg = call(k=2)
    assert rc == -2 and 'k = 1' in msg
    rc, msg = call(n_=513)
    assert rc == -2 and 'n t <= 1024' in msg
    rc, msg = call(counts=(3, 4))
    assert rc == -1 and 'add up to 7' in msg
    rc, msg = call(n_=0)
    assert rc == -1
    assert call(counts=(0, 0), rows=0)[0] == 0


def test_end_to_end_gates_and_luts(api):
    nufhe, ctx, A, B = api
    rekey = ctx.make_reencryption_key(A['sk'], B['cpk'])
    vm = B['vm']
    rng = numpy.random.RandomState(9)
    bits, mine = rng.randint(0, 2, size=(2, 4096)).astype(bool)
    moved = vm.reencrypt(rekey, ctx.encrypt(A['sk'], bits))
    assert (ctx.decrypt(B['sk'], moved) == bits).all()
    nand = vm.gate_nand(moved, ctx.encrypt(B['sk'], mine))
    assert (ctx.decrypt(B['sk'], nand) == ~(bits & mine)).all()
    # A's 2-bit LUT outputs, re-encrypted, through B's LUT
    x = rng.randint(0, 4, size=4096)
    f, g = numpy.array([3, 0, 2, 1]), numpy.array([1, 3, 0, 2])
    fa = A['vm'].lut(A['vm'].make_lut(f, 2), ctx.encrypt_int(A['sk'], x, 2))
    gb = vm.lut(vm.make_lut(g, 2), vm.reencrypt(rekey, fa))
    assert (ctx.decrypt_int(B['sk'], gb, 2) == g[f[x]]).all()


def test_multi_bit_recipient(api):
    nufhe, ctx, A, B = api
    C = _client(nufhe, ctx, multi_bit=2)
    rekey = ctx.make_reencryption_key(A['sk'], C['cpk'])
    bits = numpy.random.RandomState(10).randint(0, 2, size=4096).astype(bool)
    moved = C['vm'].reencrypt(rekey, ctx.encrypt(A['sk'], bits))
    assert (ctx.decrypt(C['sk'], moved) == bits).all()
    mine = ~bits
    assert (ctx.decrypt(C['sk'], C['vm'].gate_and(moved, ctx.encrypt(C['sk'], mine))) == (bits & mine)).all()


def _same(x, y):
    return (tuple(x.shape) == tuple(y.shape) and torch.equal(x.a, y.a) and torch.equal(x.b, y.b)
            and torch.equal(x.current_variances, y.current_variances))


@pytest.mark.parametrize('R', [None, 2])
def test_multikey_matches_per_tenant(api, R):
    nufhe, ctx, A, B = api
    sks, cks, cpks = [], [], []
    for _ in range(3):
        sk = ctx.make_secret_key()
        ck, cpk = ctx.make_cloud_key(sk, compressed=R is not None, compact_public_key=True)
        sks.append(sk), cks.append(ck), cpks.append(cpk)
    vms = [ctx.make_virtual_machine(ck.decompress(ctx.thread) if R is not None else ck) for ck in cks]
    if R is None:
        mk = ctx.make_multi_key_machine(cks + [cks[0]])
    else:
        mk = ctx.make_multi_key_machine(cks + [cks[0]], resident_tenants=R)
    rekeys = [ctx.make_reencryption_key(A['sk'], cpk) for cpk in cpks] + [None]
    sizes = [1, 1000, 2053]
    msgs = [numpy.random.RandomState(20 + t).randint(0, 2, size=s).astype(bool) for t, s in enumerate(sizes)]
    cts = [ctx.encrypt(A['sk'], m) for m in msgs] + [None]
    got = mk.reencrypt(rekeys, cts)
    assert got[3] is None
    for t in range(3):
        want = vms[t].reencrypt(rekeys[t], cts[t])
        assert _same(got[t], want), t
        assert (ctx.decrypt(sks[t], got[t]) == msgs[t]).all()


def _phase_error(thr, a, b, key, want):
    phase = thr.lwe_dot(a, key.to(a.device), add1=b, sign=-1).cpu().numpy().astype(numpy.int64)
    return ((phase - want + 2**31) % 2**32 - 2**31) / 2**32


def test_noise(api):
    """4096 re-encrypted LUT outputs and 4096 re-encrypted fresh encryptions, with the phase taken under S_B before the
    recipient's key switch and under s_B after it: every variance within 0.5 to 2 times its estimate, the mean below a
    tenth of a standard deviation from the key's offset."""
    from nufhe_b200 import reencrypt as RE, lut as L
    from nufhe_b200.lut import encode_int
    nufhe, ctx, A, B = api
    thr, p = ctx.thread, nufhe.NuFHEParameters()
    rekey = ctx.make_reencryption_key(A['sk'], B['cpk'])
    spec, body = rekey.spectra(thr)
    x = numpy.random.RandomState(11).randint(0, 4, size=4096)
    want = encode_int(x, 2).astype(numpy.int64)
    fresh = ctx.encrypt_int(A['sk'], x, 2)
    lut_out = A['vm'].lut(A['vm'].make_lut(numpy.arange(4), 2), ctx.encrypt_int(A['sk'], x, 2))
    ks = RE.keyswitch_variance(p)
    reenc = RE.reencrypt_variance(p)
    cases = [('fresh', fresh, float(fresh.current_variances[0])), ('lut', lut_out, L.bootstrap_variance(p))]
    s_b = B['sk'].lwe_key.key.reshape(-1)
    # the digits have mean -1/2, so the key's slot noises e_p leave the constant offset sum_p e_p / 2 on every result
    sample = rekey.sample.cpu().numpy().astype(numpy.int64)
    S = B['S'].cpu().numpy().astype(numpy.int64)
    slots = sample[1] - sample[0] @ compact_ref.negacyclic_matrix(S)
    msgs = numpy.zeros(N, numpy.int64)
    s_a = A['sk'].lwe_key.key.cpu().numpy().astype(numpy.int64)
    msgs[0:2 * n:2], msgs[1:2 * n:2] = s_a << 24, s_a << 16
    e = ((slots - msgs + 2**31) % 2**32 - 2**31) / 2**32
    offset = e[:2 * n].sum() / 2
    for name, ct, v_in in cases:
        ra, rb = thr.reencrypt(ct.a, ct.b, [spec], [body], [4096])
        before = _phase_error(thr, ra, rb, B['S'], want)
        out = B['vm'].reencrypt(rekey, ct)
        after = _phase_error(thr, out.a, out.b, s_b, want)
        for stage, err, est in (('before', before, v_in + reenc), ('after', after, v_in + reenc + ks)):
            var, mean = float((err**2).mean()), float(err.mean())
            print('%s, %s the key switch: variance %.4g, estimate %.4g (ratio %.3f), mean %.3g (key offset %.3g)'
                  % (name, stage, var, est, var / est, mean, offset))
            assert 0.5 * est <= var <= 2 * est
            assert abs(mean - offset) < 0.1 * est**0.5
