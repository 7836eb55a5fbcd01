"""CPU tests of the multi-key machine (nufhe_b200/multikey.py) on the oracle-backed engine double: argument validation,
idle and empty tenants, per-tenant broadcasting, and outputs equal to each tenant's own VirtualMachine."""
import ctypes

import numpy
import pytest

from multikey_fake import MultiKeyFakeEngine


class CountingEngine(MultiKeyFakeEngine):
    """Records the counts of every multi-key call."""

    def __init__(self):
        super().__init__()
        self.mk_counts = []

    def mk_bootstrap_extract(self, *args):
        self.mk_counts.append(('extract', list(args[-1])))
        return super().mk_bootstrap_extract(*args)

    def mk_keyswitch(self, keys, counts, *args, **kwds):
        self.mk_counts.append(('keyswitch', list(counts)))
        return super().mk_keyswitch(keys, counts, *args, **kwds)


@pytest.fixture(scope='module')
def mk():
    import nufhe_b200
    ctx = nufhe_b200.Context(rng=nufhe_b200.DeterministicRNG(20261017), thread=CountingEngine())
    pairs = [ctx.make_key_pair() for _ in range(3)]
    return nufhe_b200, ctx, [p[0] for p in pairs], [p[1] for p in pairs]


def _same(x, y):
    return ((x.a == y.a).all() and (x.b == y.b).all() and (x.current_variances == y.current_variances).all()
            and tuple(x.shape) == tuple(y.shape))


def test_rejects_bad_keys_and_lists(mk):
    nufhe, ctx, sks, cks = mk
    with pytest.raises(TypeError, match='tenant 1'):
        ctx.make_multi_key_machine([cks[0], 'not a key'])
    with pytest.raises(ValueError):
        ctx.make_multi_key_machine([])
    with pytest.raises(ValueError, match='tenant 0'):
        ctx.make_multi_key_machine(cks[:1], perf_params=nufhe.PerformanceParameters(cks[0].params,
                                                                                    single_kernel_bootstrap=False))
    other = nufhe.Context(rng=nufhe.DeterministicRNG(5), thread=ctx.thread).make_key_pair(tlwe_mask_size=2)[1]
    with pytest.raises(ValueError, match='tenant 1'):
        ctx.make_multi_key_machine([cks[0], other])
    machine = ctx.make_multi_key_machine(cks)
    x = ctx.encrypt(sks[0], [True])
    with pytest.raises(ValueError, match='operand 1'):
        machine.gate_nand([x, None, None], [x, None])
    with pytest.raises(ValueError, match='tenant 0'):
        machine.gate_nand([x, None, None], [None, None, None])
    with pytest.raises(TypeError):
        machine.gate_nand([x, None, None])
    with pytest.raises(AttributeError):
        machine.gate_frobnicate([x, None, None])
    with pytest.raises(ValueError, match='dest'):
        machine.gate_nand([x, None, None], [x, None, None], dest=[None])
    with pytest.raises(ValueError):
        machine.lut(ctx.make_virtual_machine(cks[0]).make_lut(numpy.zeros((2, 4), int), bits=2, log2_outputs=0),
                    [x, None, None])


def test_rejects_multibit_key(mk):
    nufhe, ctx, sks, cks = mk
    ck2 = ctx.make_cloud_key(sks[0], multi_bit=2)
    with pytest.raises(ValueError, match='tenant 1.*multi-bit'):
        ctx.make_multi_key_machine([cks[0], ck2])


def test_gates_equal_per_tenant_machines(mk):
    nufhe, ctx, sks, cks = mk
    # a repeated key, an idle tenant and per-tenant broadcasting (tenant 0: (2, 3) with (3,), tenant 3: (1,) with (2,))
    keys = [cks[0], cks[1], cks[2], cks[0]]
    secrets = [sks[0], sks[1], sks[2], sks[0]]
    machine = ctx.make_multi_key_machine(keys)
    rng = numpy.random.RandomState(3)
    shapes = [((2, 3), (3,)), None, ((4,), (4,)), ((1,), (2,))]
    bits = [None if s is None else (rng.randint(0, 2, s[0]).astype(bool), rng.randint(0, 2, s[1]).astype(bool))
            for s in shapes]
    xs = [None if b is None else ctx.encrypt(secrets[t], b[0]) for t, b in enumerate(bits)]
    ys = [None if b is None else ctx.encrypt(secrets[t], b[1]) for t, b in enumerate(bits)]
    thr = ctx.thread
    thr.mk_counts.clear()
    out = machine.gate_nand(xs, ys)
    assert thr.mk_counts == [('extract', [6, 0, 4, 2]), ('keyswitch', [6, 0, 4, 2])]
    assert out[1] is None
    for t in (0, 2, 3):
        want = ctx.make_virtual_machine(keys[t]).gate_nand(xs[t], ys[t])
        assert _same(out[t], want), t
        assert (ctx.decrypt(secrets[t], out[t]) == ~(bits[t][0] & bits[t][1])).all()
    # MUX with dest, and the keyless gates
    zs = [None if b is None else ctx.encrypt(secrets[t], ~b[1]) for t, b in enumerate(bits)]
    dest = [None if x is None else machine.empty_ciphertext(out[t].shape) for t, x in enumerate(xs)]
    res = machine.gate_mux(xs, ys, zs, dest=dest)
    for t in (0, 2, 3):
        assert res[t] is dest[t]
        assert _same(res[t], ctx.make_virtual_machine(keys[t]).gate_mux(xs[t], ys[t], zs[t])), t
    nots = machine.gate_not(xs)
    consts = machine.gate_constant([[True, False], None, None, [True]])
    assert (ctx.decrypt(secrets[0], nots[0]) == ~bits[0][0]).all() and nots[1] is None
    assert (ctx.decrypt(secrets[3], consts[3]) == [True]).all() and consts[2] is None


def test_lut_equals_per_tenant_machines(mk):
    nufhe, ctx, sks, cks = mk
    machine = ctx.make_multi_key_machine(cks)
    vms = [ctx.make_virtual_machine(ck) for ck in cks]
    adder = vms[0].make_lut([[v % 2 for v in range(4)], [v // 2 for v in range(4)]], bits=2)
    vals = [numpy.array([1, 3]), numpy.array([2]), None]
    xs = [None if v is None else ctx.encrypt_int(sks[t], v, 2) for t, v in enumerate(vals)]
    out = machine.lut(adder, xs)
    assert out[2] is None
    for t in (0, 1):
        want = vms[t].lut(adder, xs[t])
        assert len(out[t]) == 2 and all(_same(o, w) for o, w in zip(out[t], want)), t
        assert (ctx.decrypt_int(sks[t], out[t][1], 2) == vals[t] // 2).all()
    # two inputs, one output
    t2 = vms[0].make_lut([0, 1, 0, 0], bits=2, out='bool')
    ys = [None if v is None else ctx.encrypt_int(sks[t], 1 - v % 2, 2) for t, v in enumerate(vals)]
    out = machine.lut(t2, xs, ys)
    for t in (0, 1):
        assert _same(out[t], vms[t].lut(t2, xs[t], ys[t])), t
    with pytest.raises(ValueError):
        machine.lut(vms[0].make_lut([0, 1, 2, 3], bits=2), xs, ys, shift=2)


def test_all_tenants_idle(mk):
    nufhe, ctx, sks, cks = mk
    machine = ctx.make_multi_key_machine(cks[:2])
    assert machine.gate_xor([None, None], [None, None]) == [None, None]


def test_capi_multikey_entry_points_reject_a_null_context():
    from nufhe_b200 import _native
    lib = _native.load()
    keys = (ctypes.c_void_p * 1)(None)
    counts = (ctypes.c_size_t * 1)(0)
    assert lib.nb_mk_bootstrap_extract(None, None, None, None, None, 0, 1, 1, 1, keys, counts, 1, 500, None, None,
                                       0) == _native.NB_EINVAL
    assert lib.nb_mk_keyswitch(None, None, None, None, None, 0, keys, keys, keys, counts, 1, 1024, 500, 8, 2, None,
                               None, None, 0) == _native.NB_EINVAL
