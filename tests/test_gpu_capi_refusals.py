"""Argument checks of the C entry points: each call below must be refused by host code with its return code and its
exact nb_last_error text, or be an empty batch, before anything is launched.

Pointers that must be non-null point into one small valid device buffer; no case reaches a kernel.  The two empty-batch
rules of the bootstraps are pinned too: a single-key call returns NB_OK at batch 0 before any check, a multi-key call
checks its counts and every tenant's key even at batch 0 (MultiKeyVirtualMachine validates its keys that way)."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu
N = 1024
OK, EINVAL, EUNSUPPORTED = 0, -1, -2


@pytest.fixture(scope='module')
def eng():
    from nufhe_b200.engine import Engine
    return Engine(0)


@pytest.fixture(scope='module')
def buf(eng):
    return eng.empty((1 << 16,), torch.int32)


@pytest.fixture(scope='module')
def key(eng):
    """A prepared engine key of 2 rows (all zero: integral, so it carries FP64 spectra): a valid key of every tenant."""
    return eng.bk_prepare(torch.zeros((2 * 8 * N,), dtype=torch.int64, device=eng.device))


def ptrs(ctype, values):
    return (ctype * max(len(values), 1))(*values)


def sizes(values):
    return ptrs(ctypes.c_size_t, values)


def keys(values):
    return ptrs(ctypes.c_void_p, values)


def ids(values):
    return ptrs(ctypes.c_uint32, values)


@pytest.fixture
def refused(eng):
    def check(rc, code, text):
        assert rc == code, (rc, eng.lib.nb_last_error(eng.handle).decode())
        assert eng.lib.nb_last_error(eng.handle).decode() == text
    return check


def test_bootstraps(eng, buf, refused):
    lib, h, p = eng.lib, eng.handle, buf.data_ptr()
    refused(lib.nb_bootstrap_extract(h, None, p, None, None, 0, 1, 0, 0, p, 500, p, p, 2), EINVAL,
            'nb_bootstrap_extract: null argument')
    refused(lib.nb_bootstrap_extract(h, p, p, p, None, 0, 1, 1, 0, p, 500, p, p, 2), EINVAL,
            'nb_bootstrap_extract: in2_a/in2_b must come together')
    refused(lib.nb_bootstrap_extract(h, p, p, None, None, 0, 1, 0, 0, p, 0, p, p, 2), EUNSUPPORTED,
            'LWE dimension out of range')
    refused(lib.nb_bootstrap_lut_extract(h, p, p, None, None, 0, 1, 0, None, 0, 0, p, 500, p, p, 2), EINVAL,
            'nb_bootstrap_lut_extract: null argument')
    refused(lib.nb_bootstrap_lut_extract(h, p, p, None, p, 0, 1, 1, p, 0, 0, p, 500, p, p, 2), EINVAL,
            'nb_bootstrap_lut_extract: in2_a/in2_b must come together')
    refused(lib.nb_bootstrap_lut_extract(h, p, p, None, None, 0, 1, 0, p, 7, 0, p, 500, p, p, 2), EINVAL,
            'nb_bootstrap_lut_extract: tv_stride must be 0 or 1024')
    refused(lib.nb_bootstrap_lut_extract(h, p, p, None, None, 0, 1, 0, p, 0, 3, p, 500, p, p, 2), EINVAL,
            'nb_bootstrap_lut_extract: log2_outputs must be 0, 1 or 2')
    refused(lib.nb_bootstrap_lut_extract(h, p, p, None, None, 0, 1, 0, p, N, -1, p, 500, p, p, 2), EINVAL,
            'nb_bootstrap_lut_extract: log2_outputs must be 0, 1 or 2')
    refused(lib.nb_bootstrap_glwe_lut_extract(h, p, p, None, p, 500, p, p, 2), EINVAL,
            'nb_bootstrap_glwe_lut_extract: null argument')
    refused(lib.nb_bootstrap_glwe_lut_extract(h, p, p, p, None, 500, p, p, 2), EINVAL,
            'nb_bootstrap_glwe_lut_extract: null argument')
    refused(lib.nb_bootstrap_extract2(h, p, p, None, None, 0, 1, 0, None, p, None, None, 0, 1, 0, 0, p, 500, p, p, 2),
            EINVAL, 'nb_bootstrap_extract2: null argument')
    refused(lib.nb_bootstrap_extract2(h, p, p, None, None, 0, 1, 0, p, p, p, None, 0, 1, 1, 0, p, 500, p, p, 2),
            EINVAL, 'nb_bootstrap_extract2: a/b parts must come together')
    refused(lib.nb_bootstrap_extract2(h, p, p, None, p, 0, 1, 1, p, p, None, None, 0, 1, 0, 0, p, 500, p, p, 2),
            EINVAL, 'nb_bootstrap_extract2: a/b parts must come together')


def test_bootstraps_single_key_empty_batch(eng, refused):
    """batch 0 returns NB_OK before any check: null operands, null key and a bad n or test-vector layout pass."""
    lib, h = eng.lib, eng.handle
    assert lib.nb_bootstrap_extract(h, None, None, None, None, 0, 1, 0, 0, None, 0, None, None, 0) == OK
    assert lib.nb_bootstrap_lut_extract(h, None, None, None, None, 0, 1, 0, None, 7, 3, None, 0, None, None, 0) == OK
    assert lib.nb_bootstrap_glwe_lut_extract(h, None, None, None, None, 0, None, None, 0) == OK
    assert lib.nb_bootstrap_extract2(h, None, None, None, None, 0, 1, 0, None, None, None, None, 0, 1, 0, 0, None, 0,
                                     None, None, 0) == OK


def _mk_calls(lib, h, p):
    """The four multi-key bootstraps over a batch of `b` ciphertexts of `n` = 2 with the given keys and counts."""
    return {
        'nb_mk_bootstrap_extract': lambda k, c, t, b, n=2: lib.nb_mk_bootstrap_extract(
            h, p, p, None, None, 0, 1, 0, 0, k, c, t, n, p, p, b),
        'nb_mk_bootstrap_extract2': lambda k, c, t, b, n=2: lib.nb_mk_bootstrap_extract2(
            h, p, p, None, None, 0, 1, 0, p, p, None, None, 0, 1, 0, 0, k, c, t, n, p, p, b),
        'nb_mk_bootstrap_lut_extract': lambda k, c, t, b, n=2: lib.nb_mk_bootstrap_lut_extract(
            h, p, p, None, None, 0, 1, 0, p, 0, 0, k, c, t, n, p, p, b),
        'nb_mk_bootstrap_glwe_lut_extract': lambda k, c, t, b, n=2: lib.nb_mk_bootstrap_glwe_lut_extract(
            h, p, p, p, k, c, t, n, p, p, b),
    }


def test_multikey_bootstraps(eng, buf, key, refused):
    lib, h, p, k = eng.lib, eng.handle, buf.data_ptr(), key.data_ptr()
    for name, call in _mk_calls(lib, h, p).items():
        refused(call(None, sizes([2]), 1, 2), EINVAL, name + ': null argument')
        refused(call(keys([k]), None, 1, 2), EINVAL, name + ': null argument')
        refused(call(keys([k, k]), sizes([1, 0]), 2, 2), EINVAL, name + ': the counts add up to 1, not the batch 2')
        refused(call(keys([k, None]), sizes([1, 1]), 2, 2), EINVAL, name + ': null key of tenant 1')
        refused(call(keys([k, p]), sizes([1, 1]), 2, 2), EINVAL,
                name + ': the key of tenant 1 is not inside an engine key with FP64 spectra prepared on this context or '
                       'a slot filled by nb_mk_bk_expand')
        refused(call(keys([k, k]), sizes([1, 1]), 2, 2, n=0), EUNSUPPORTED, name + ': LWE dimension out of range')
    refused(lib.nb_mk_bootstrap_extract(h, None, p, None, None, 0, 1, 0, 0, keys([k]), sizes([2]), 1, 2, p, p, 2),
            EINVAL, 'nb_mk_bootstrap_extract: null argument')
    refused(lib.nb_mk_bootstrap_extract(h, p, p, p, None, 0, 1, 1, 0, keys([k]), sizes([2]), 1, 2, p, p, 2),
            EINVAL, 'nb_mk_bootstrap_extract: in2_a/in2_b must come together')
    refused(lib.nb_mk_bootstrap_extract2(h, p, p, None, None, 0, 1, 0, p, p, None, p, 0, 1, 1, 0, keys([k]), sizes([2]),
                                         1, 2, p, p, 2), EINVAL, 'nb_mk_bootstrap_extract2: a/b parts must come together')
    refused(lib.nb_mk_bootstrap_lut_extract(h, p, p, None, None, 0, 1, 0, None, 0, 0, keys([k]), sizes([2]), 1, 2, p,
                                            p, 2), EINVAL, 'nb_mk_bootstrap_lut_extract: null argument')
    refused(lib.nb_mk_bootstrap_lut_extract(h, p, p, None, p, 0, 1, 1, p, 0, 0, keys([k]), sizes([2]), 1, 2, p, p, 2),
            EINVAL, 'nb_mk_bootstrap_lut_extract: in2_a/in2_b must come together')
    refused(lib.nb_mk_bootstrap_lut_extract(h, p, p, None, None, 0, 1, 0, p, 2 * N, 0, keys([k]), sizes([2]), 1, 2, p,
                                            p, 2), EINVAL, 'nb_mk_bootstrap_lut_extract: tv_stride must be 0 or 1024')
    refused(lib.nb_mk_bootstrap_lut_extract(h, p, p, None, None, 0, 1, 0, p, 0, 3, keys([k]), sizes([2]), 1, 2, p, p, 2),
            EINVAL, 'nb_mk_bootstrap_lut_extract: log2_outputs must be 0, 1 or 2')
    refused(lib.nb_mk_bootstrap_glwe_lut_extract(h, p, p, None, keys([k]), sizes([2]), 1, 2, p, p, 2), EINVAL,
            'nb_mk_bootstrap_glwe_lut_extract: null argument')


def test_multikey_bootstraps_empty_batch(eng, buf, key, refused):
    """batch 0 still checks the counts and every tenant's key (null operands are allowed), and passes when they hold."""
    lib, h, p, k = eng.lib, eng.handle, buf.data_ptr(), key.data_ptr()
    for name, call in _mk_calls(lib, h, None).items():
        refused(call(keys([k]), sizes([1]), 1, 0), EINVAL, name + ': the counts add up to 1, not the batch 0')
        refused(call(keys([k, None]), sizes([0, 0]), 2, 0), EINVAL, name + ': null key of tenant 1')
        refused(call(keys([k, p]), sizes([0, 0]), 2, 0), EINVAL,
                name + ': the key of tenant 1 is not inside an engine key with FP64 spectra prepared on this context or '
                       'a slot filled by nb_mk_bk_expand')
        assert call(keys([k, k]), sizes([0, 0]), 2, 0) == OK
        assert call(None, None, 0, 0) == OK


def test_keyswitches(eng, buf, refused):
    lib, h, p = eng.lib, eng.handle, buf.data_ptr()

    def ks(src1_a=p, src2_a=None, src2_b=None, ks_a=p, in_size=1024, n=500, t=8, log2_base=2, batch=2):
        return lib.nb_keyswitch(h, src1_a, p, src2_a, src2_b, 0, ks_a, p, p, in_size, n, t, log2_base, p, p, None, batch)
    refused(ks(src1_a=None), EINVAL, 'nb_keyswitch: null argument')
    refused(ks(ks_a=None), EINVAL, 'nb_keyswitch: null argument')
    refused(ks(src2_a=p), EINVAL, 'nb_keyswitch: src2_a/src2_b must come together')
    refused(ks(n=600), EUNSUPPORTED, 'nb_keyswitch: output LWE dimension above 511')
    refused(ks(t=0), EINVAL, 'nb_keyswitch: bad decomposition')
    refused(ks(t=8, log2_base=4), EINVAL, 'nb_keyswitch: bad decomposition')
    assert ks(src1_a=None, ks_a=None, n=600, t=0, batch=0) == OK

    def mk(ks_a=(p, p), ks_b=(p, p), ks_cv=(p, p), counts=(1, 1), tenants=2, src1_a=p, src2_b=None, in_size=1024, n=500,
           t=8, batch=2):
        return lib.nb_mk_keyswitch(h, src1_a, p, None, src2_b, 0, ks_a and keys(ks_a), ks_b and keys(ks_b),
                                   ks_cv and keys(ks_cv), counts and sizes(counts), tenants, in_size, n, t, 2, p, p, None,
                                   batch)
    refused(mk(ks_cv=None), EINVAL, 'nb_mk_keyswitch: null argument')
    refused(mk(counts=None), EINVAL, 'nb_mk_keyswitch: null argument')
    refused(mk(counts=(2, 1)), EINVAL, 'nb_mk_keyswitch: the counts add up to 3, not the batch 2')
    refused(mk(src1_a=None), EINVAL, 'nb_mk_keyswitch: null argument')
    refused(mk(src2_b=p), EINVAL, 'nb_mk_keyswitch: src2_a/src2_b must come together')
    refused(mk(ks_b=(p, None)), EINVAL, 'nb_mk_keyswitch: null key of tenant 1')
    refused(mk(ks_cv=(p, None)), EINVAL, 'nb_mk_keyswitch: null key of tenant 1')
    for shape in ({'in_size': 512}, {'n': 630}, {'t': 3}):
        refused(mk(**shape), EUNSUPPORTED,
                'nb_mk_keyswitch: the grouped key switch is for in = 1024, n = 500, t = 8, base 4 only')
    refused(mk(ks_a=(p, None), counts=(0, 0), src1_a=None, batch=0), EINVAL, 'nb_mk_keyswitch: null key of tenant 1')
    assert mk(counts=(0, 0), src1_a=None, batch=0) == OK


def test_multikey_gemms_and_expansions(eng, buf, refused):
    lib, h, p = eng.lib, eng.handle, buf.data_ptr()
    tree = lambda planes, counts, tenants=2, rows=2, n=500, k=1, a=p: lib.nb_mk_tree_keyswitch(  # noqa: E731
        h, a, planes, counts, tenants, n, k, p, rows)
    refused(tree(None, sizes([1, 1])), EINVAL, 'nb_mk_tree_keyswitch: null argument')
    refused(tree(keys([p, p]), sizes([2, 1])), EINVAL, 'nb_mk_tree_keyswitch: the counts add up to 3, not the batch 2')
    refused(tree(keys([p, p]), sizes([1, 1]), a=None), EINVAL, 'nb_mk_tree_keyswitch: null argument')
    refused(tree(keys([p, None]), sizes([1, 1])), EINVAL, 'nb_mk_tree_keyswitch: null planes of tenant 1')
    refused(tree(keys([p, p]), sizes([1, 1]), k=0), EINVAL, 'nb_mk_tree_keyswitch: bad mask size')

    mac = lambda key, counts, tenants=2, groups=2, rows=4, outs=2, x=p: lib.nb_mk_ntt_mac(  # noqa: E731
        h, x, key, counts, tenants, p, rows, outs, groups)
    refused(mac(keys([p, p]), None), EINVAL, 'nb_mk_ntt_mac: null argument')
    refused(mac(keys([p, p]), sizes([0, 1])), EINVAL, 'nb_mk_ntt_mac: the counts add up to 1, not the batch 2')
    refused(mac(keys([p, None]), sizes([1, 1])), EINVAL, 'nb_mk_ntt_mac: null key of tenant 1')
    refused(mac(keys([p, p]), sizes([1, 1]), rows=0), EINVAL,
            'nb_mk_ntt_mac: rows must be in [1, 2^24] and outputs in [1, 2^16]')

    seeds = (ctypes.c_uint32 * 16)()
    bk = lambda bodies, slots, n=2, k=1: lib.nb_mk_bk_expand(h, seeds, bodies, slots, 2, n, k, 2, N)  # noqa: E731
    refused(bk(None, keys([p, p])), EINVAL, 'nb_mk_bk_expand: null argument')
    refused(bk(keys([p, p]), keys([p, None])), EINVAL, 'nb_mk_bk_expand: null bodies or slot of tenant 1')
    refused(bk(keys([p, None]), keys([p, p])), EINVAL, 'nb_mk_bk_expand: null bodies or slot of tenant 1')
    refused(bk(keys([p, p]), keys([p, p]), k=2), EUNSUPPORTED,
            'nb_mk_bk_expand: the expansion is for k = 1, l = 2, N = 1024 and 1 <= n <= 1024 only')

    ks = lambda ks_a, n=500: lib.nb_mk_ks_expand(h, seeds, ks_a, 2, 1024, 8, 2, n)  # noqa: E731
    refused(ks(None), EINVAL, 'nb_mk_ks_expand: null argument')
    refused(ks(keys([p, None])), EINVAL, 'nb_mk_ks_expand: null ks_a of tenant 1')
    refused(ks(keys([p, p]), n=499), EUNSUPPORTED,
            'nb_mk_ks_expand: the expansion is for the multi-key key switch, in = 1024, n = 500, t = 8, base 4 only')


def test_index_calls(eng, buf, refused):
    lib, h, p = eng.lib, eng.handle, buf.data_ptr()
    bits_text = ': bits must be 1 to 20'
    cols_text = ': columns * 2^bits must be at most N below 10 bits'

    refused(lib.nb_index_cmux_level(h, p, 0, None, 0, p, 1, 2), EINVAL, 'nb_index_cmux_level: null argument')

    rot = lambda bits, columns, acc=p: lib.nb_index_rotate_extract(h, acc, 0, p, 0, bits, columns, p, p, 2)  # noqa: E731
    refused(rot(3, 1, acc=None), EINVAL, 'nb_index_rotate_extract: null argument')
    for bits, columns, text in ((0, 1, bits_text), (21, 1, bits_text), (5, 64, cols_text), (9, 3, cols_text),
                                (4, 0, cols_text)):
        refused(rot(bits, columns), EINVAL, 'nb_index_rotate_extract' + text)

    def rot_ind(bits, columns, stride=2 * N, table_ids=(0, 1), count=2, tables=p):
        return lib.nb_index_rotate_extract_indirect(h, tables, stride, count, ids(table_ids), p, 0, bits, columns, p, p,
                                                    len(table_ids))
    what = 'nb_index_rotate_extract_indirect'
    refused(rot_ind(3, 1, tables=None), EINVAL, what + ': null argument')
    for bits, columns, text in ((0, 1, bits_text), (21, 1, bits_text), (5, 64, cols_text)):
        refused(rot_ind(bits, columns), EINVAL, what + text)
    refused(rot_ind(3, 1, stride=2 * N - 1), EINVAL, what + ': tables overlap')
    refused(rot_ind(12, 2, stride=2 * N), EINVAL, what + ': tables overlap')
    refused(rot_ind(3, 1, table_ids=(0, 2)), EINVAL, what + ': query 1 names table 2 of 2')

    def cmux_ind(stride=4 * N, table_ids=(1, 0), count=2, nodes=1, tables=p):
        return lib.nb_index_cmux_level_indirect(h, tables, stride, count, ids(table_ids), p, 0, p, nodes, len(table_ids))
    what = 'nb_index_cmux_level_indirect'
    refused(cmux_ind(tables=None), EINVAL, what + ': null argument')
    refused(cmux_ind(stride=4 * N - 2), EINVAL, what + ': tables overlap')
    refused(cmux_ind(stride=4 * N, nodes=2), EINVAL, what + ': tables overlap')
    refused(cmux_ind(table_ids=(5, 0)), EINVAL, what + ': query 0 names table 5 of 2')
    refused(cmux_ind(table_ids=(0, 1, 2), count=2), EINVAL, what + ': query 2 names table 2 of 2')

    asm = lambda bits, columns, b=p: lib.nb_index_write_assemble(h, None, b, bits, columns, p, 2)  # noqa: E731
    refused(asm(3, 1, b=None), EINVAL, 'nb_index_write_assemble: null argument')
    for bits, columns, text in ((0, 1, bits_text), (21, 1, bits_text), (5, 64, cols_text)):
        refused(asm(bits, columns), EINVAL, 'nb_index_write_assemble' + text)

    def wrot(bits, columns, acc=p, stride=2 * N, count=1, table_ids=None, delta=p):
        return lib.nb_index_write_rotate(h, delta, p, 0, bits, columns, p if acc is None else None, acc, stride, count,
                                         table_ids and ids(table_ids), 2)
    what = 'nb_index_write_rotate'
    for bits, columns, text in ((0, 1, bits_text), (21, 1, bits_text), (5, 64, cols_text)):
        refused(wrot(bits, columns), EINVAL, what + text)
    refused(wrot(12, 1), EINVAL, what + ': the rotation adds into the tables exactly when bits <= 10')
    refused(wrot(3, 1, acc=None), EINVAL, what + ': the rotation adds into the tables exactly when bits <= 10')
    refused(wrot(3, 1, delta=None), EINVAL, what + ': null argument')
    refused(wrot(3, 1, stride=2 * N - 1), EINVAL, what + ': the tables overlap or are not named per query')
    refused(wrot(3, 1, count=2), EINVAL, what + ': the tables overlap or are not named per query')
    refused(wrot(3, 1, count=2, table_ids=(1, 2)), EINVAL, what + ': query 1 names table 2 of 2')

    def demux(acc=p, stride=4 * N, count=1, table_ids=None, nodes=1, sel=p):
        return lib.nb_index_demux_level(h, p, sel, 0, p, acc, stride, count, table_ids and ids(table_ids), nodes, 2)
    what = 'nb_index_demux_level'
    refused(demux(sel=None), EINVAL, what + ': null argument')
    refused(demux(stride=4 * N - 1), EINVAL, what + ': the tables overlap or are not named per query')
    refused(demux(count=0), EINVAL, what + ': the tables overlap or are not named per query')
    refused(demux(count=3, table_ids=(0, 3)), EINVAL, what + ': query 1 names table 3 of 3')
