"""CPU checks of the multi-key matrix's infrastructure (tests/mk_ref.py): its restatements of the tile and group tables
equal the library's own (csrc/mk_layout.cuh through the host emulator), its key-switch band builder reaches the tile
counts and splits it promises, and its per-tenant compositions equal the oracle on every tenant's segment."""
import ctypes
import os

import numpy
import pytest

import fused_ref as F
import gen_inputs as G
import mk_ref as MK
from oracle import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 1024
EDGE_MIXES = [(0,), (1,), (255,), (256,), (257,), (0, 0), (0, 1, 255, 256, 257, 0), (513, 2, 0, 700), (1,) * 300,
              (0, 1, 2, 0, 3), (511, 0, 0, 512, 1)]


@pytest.fixture(scope='module')
def emul():
    path = os.path.join(ROOT, 'nufhe_b200', 'csrc', 'libnb_host_emul.so')
    if not os.path.exists(path):
        import __graft_entry__ as g
        g.build()
    lib = ctypes.CDLL(path)
    lib.emul_mk_tree_tiles.restype = ctypes.c_uint64
    lib.emul_mk_tree_tiles.argtypes = [ctypes.c_void_p, ctypes.c_size_t] + [ctypes.c_void_p] * 3
    lib.emul_mk_group_tenants.restype = ctypes.c_uint64
    lib.emul_mk_group_tenants.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    return lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


@pytest.mark.parametrize('counts', EDGE_MIXES)
def test_tree_tiles_equal_the_library(emul, counts):
    c = numpy.asarray(counts, numpy.uintp)
    n = emul.emul_mk_tree_tiles(_p(c), len(counts), None, None, None)
    row0, rows, tenant = numpy.zeros(n, numpy.uint64), numpy.zeros(n, numpy.uint32), numpy.zeros(n, numpy.uint32)
    emul.emul_mk_tree_tiles(_p(c), len(counts), _p(row0), _p(rows), _p(tenant))
    assert list(zip(row0.tolist(), rows.tolist(), tenant.tolist())) == MK.tree_tiles(counts)


@pytest.mark.parametrize('counts', EDGE_MIXES)
def test_group_tenants_equal_the_library(emul, counts):
    owner = numpy.full(sum(counts), 0xdead, numpy.uint32)
    assert emul.emul_mk_group_tenants(_p(numpy.asarray(counts, numpy.uintp)), len(counts), _p(owner)) == sum(counts)
    assert (owner == MK.group_tenants(counts)).all()


def test_tenant_of_and_truncate():
    assert MK.tenant_of([2, 0, 1]).tolist() == [0, 0, 2]
    assert MK.tenant_of([2, 0, 1], jobs=2).tolist() == [0, 0, 2, 0, 0, 2]
    assert MK.truncate([0, 3, 1, 0, 2], 4) == [0, 3, 1, 0, 0]
    assert MK.truncate([0, 3, 1, 0, 2], 2) == [0, 2, 0, 0, 0]
    for counts in EDGE_MIXES:
        for B in {0, min(1, sum(counts)), sum(counts) // 2, sum(counts)}:
            assert (MK.tenant_of(MK.truncate(counts, B)) == MK.tenant_of(counts)[:B]).all()


@pytest.mark.parametrize('counts', EDGE_MIXES + [(31, 32, 33), (4096, 1, 3)])
def test_keyswitch_tiles_never_cross_a_tenant(counts):
    owner = MK.tenant_of(counts)
    covered = numpy.zeros(sum(counts), int)
    for t, r0, r in MK.ks_tiles(counts):
        assert 1 <= r <= MK.KS_TILE and (owner[r0:r0 + r] == t).all()
        covered[r0:r0 + r] += 1
    assert (covered == 1).all()
    # a GEMM tenant's rows are in no tile; a registered tenant below the threshold keeps its tiles
    assert MK.ks_gemm_tenants([31, 64, 63, 64], {1, 2}, 64) == [1]
    assert [t for t, _, _ in MK.ks_tiles([31, 64, 63, 64], {1, 2}, 64)] == [0, 2, 2, 3, 3]


@pytest.mark.parametrize('sm', [132, 114, 78])
def test_band_builder(sm):
    """every mix of ks_band_mixes has the tile count of a band edge and that band's split; the tile count one below a
    band's first edge (one above its last) gives another split; every split band is reached"""
    bands = MK.ks_split_bands(sm)
    seen = set()
    for s, counts in MK.ks_band_mixes(sm):
        tiles = len(MK.ks_tiles(counts))
        lo, hi = bands[s]
        assert tiles in (lo, hi if hi is not None else lo + 1), (sm, s, tiles)
        assert MK.ks_splits(tiles, sm) == s
        if tiles == lo and lo > 1:
            assert MK.ks_splits(lo - 1, sm) != s
        if hi is not None and tiles == hi:
            assert MK.ks_splits(hi + 1, sm) != s
        assert all(1 <= c <= 33 for c in counts)
        seen.add(s)
    assert seen == set(bands)
    assert bands[min(MK.KS_MAX_SPLITS, sm)][0] == 1 and bands[1][1] is None
    assert any(31 in c and 32 in c and 33 in c for _, c in MK.ks_band_mixes(sm))


# ---- the per-tenant compositions ------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def small_keys():
    """three random integral keys of 6 rows in the reference's form"""
    rng = G.rs(4000)
    return [O.bk_transform(G.torus32(rng, (6, 2, 2, 2, N))) for _ in range(3)]


def _modes(bks, counts, ref, B):
    n, t = 6, O.phase_to_t32
    return [F.gate_mode('nand', n, bks, t(1, 8), -1, -1, 2**29, True, 4001, B, ref=ref),
            F.x2_mode('x2', n, bks, (t(-1, 8), 1, 1, True), (-55555, 3, 7, False), 2**29, 4002, B, ref=ref),
            F.lut_mode('lut', n, bks, 2, True, True, 4003, B, ref=ref),
            F.lut_mode('lut_shared', n, bks, 1, False, False, 4004, B, ref=ref),
            F.glwe_mode('glwe', n, bks, 4005, B, ref=ref)]


def test_one_tenant_equals_the_standard_composition(small_keys):
    B = 5
    got = _modes([small_keys[1]], [B], MK.ref(MK.tenant_of([B])), B)
    want = _modes(small_keys[1], [B], F.STANDARD, B)
    for g, w in zip(got, want):
        assert all((x == y).all() for x, y in zip(g.want, w.want)), g.name


def test_two_tenants_equal_the_oracle_on_each_segment(small_keys):
    """counts (3, 4) with different keys: each tenant's rows equal the oracle's composition with that tenant's key,
    and differ from the other key's"""
    counts = [3, 4]
    B = sum(counts)
    got = _modes(small_keys[:2], counts, MK.ref(MK.tenant_of(counts)), B)
    for t, lo, hi in MK.segments(counts):
        for other in range(2):
            want = _modes(small_keys[other], counts, F.STANDARD, B)
            for g, w in zip(got, want):
                same = all((x[lo:hi] == y[lo:hi]).all() for x, y in zip(g.want, w.want))
                assert same == (other == t), (g.name, t, other)
    # the gate rows also equal the oracle's bootstrap taken directly on the segment
    nand = got[0]
    x1, x2 = F.lwe_inputs(G.rs(4001), B, 6, O.phase_to_t32(1, 8), -1, -1, True, F.gate_targets())
    for t, lo, hi in MK.segments(counts):
        a, b = F.prologue((x1[0][lo:hi], x1[1][lo:hi]), (x2[0][lo:hi], x2[1][lo:hi]), O.phase_to_t32(1, 8), -1, -1)
        wa, wb = O.bootstrap(a, b, small_keys[t], None, 2**29)
        assert (nand.want[0][lo:hi] == wa).all() and (nand.want[1][lo:hi] == wb).all(), t
