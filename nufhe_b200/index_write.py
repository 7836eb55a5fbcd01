"""Oblivious writes into encrypted tables (DESIGN.md section 21): add to, or overwrite, the entry at a client-encrypted
index of an EncryptedIndexTable, without the server learning which entry changed.

A write is the transpose of a lookup (index_lookup.py) on the same selectors and the same FP64 CMux step:
  * the delta of query q is one GLWE sample under S per accumulator, (0, b) - V, V the tree key switch of the value's
    mask (nothing for plain values); for m < 10 column w sits at coefficient w 2^m (nb_index_write_assemble);
  * for j < min(m, 10), ACC <- ACC + C_j [x] ((X^(+2^j) - 1) ACC), which leaves X^(idx mod 1024) D
    (nb_index_write_rotate);
  * for j = m-1 down to 10, node y becomes (y - C_j [x] y, C_j [x] y) (nb_index_demux_level), which sends the delta to
    the leaf that holds the entry and leaves a small noise in every other leaf;
  * the last level adds every leaf into an int32 copy of the table's nodes (red.global.add: sums mod 2^32 do not depend
    on the order of the adds), which is rounded to the 16-bit wire form once per call.
Every call changes every entry's ciphertext, and its work is the same for every index.  Noise: index_lookup's
write_variance and written_table_variance; a call that would leave the table below lut.MARGIN_SIGMAS on its lookups
raises ValueError, and refresh_table resets the noise with one bootstrap per entry.
"""
import numpy
import torch

from .lwe import LweSampleArray
from .gates import MU
from .batch_keys import OneKey
from .index_lookup import (EncryptedIndexArray, CompressedEncryptedIndexArray, EncryptedIndexTable, IndexTable, N,
                           ROTATE_BITS, selector_passes, _round16, _wrap32, lookup, keyswitch_variance,
                           written_table_variance, check_table_variance, make_encrypted_table)


def check_arguments(what, params, index, table, tree_key, values):
    """The checks lookup makes, and those of the values: TypeError for a compressed index, a table of another kind or
    anything but a NuFHETreeKey with LWE values; ValueError for other parameters or another bit count."""
    from .tree_lut import NuFHETreeKey
    if not isinstance(index, EncryptedIndexArray):
        raise TypeError('%s needs an EncryptedIndexArray%s, got %s'
                        % (what, ' (decompress() it first)' if isinstance(index, CompressedEncryptedIndexArray) else '',
                           type(index).__name__))
    if not isinstance(table, (IndexTable, EncryptedIndexTable)):
        raise TypeError('%s needs an EncryptedIndexTable or an IndexTable, got %s' % (what, type(table).__name__))
    if index.params != params or table.params != params:
        raise ValueError('the encrypted index or the table was made for other parameters than this machine')
    if index.bits != table.bits:
        raise ValueError('the table takes %d-bit indices, got %d bits' % (table.bits, index.bits))
    lwe = isinstance(values, LweSampleArray) or (isinstance(values, (list, tuple)) and len(values) > 0
                                                 and isinstance(values[0], LweSampleArray))
    if lwe or tree_key is not None:
        if not isinstance(tree_key, NuFHETreeKey):
            raise TypeError('%s of ciphertexts needs a NuFHETreeKey (ctx.make_cloud_key(sk, tree_key=True)), got %s'
                            % (what, type(tree_key).__name__))
        if tree_key.params != params:
            raise ValueError('the tree key was made for other parameters than this machine')
    return lwe


def table_nodes(table):
    """An int32 copy of the table's nodes (P, 2, N), the accumulator of a write: an IndexTable is the noiseless
    trivial encryption of its entries."""
    return (table.nodes if isinstance(table, EncryptedIndexTable) else table.polys).clone()


def leaf_variance(table):
    return table.variance if isinstance(table, EncryptedIndexTable) else 0.0


def lwe_values(params, shape, W, values):
    """a (B, W, n), b (B, W) int32 and the per-query variances of LWE values: an LweSampleArray (W = 1) or a list of W,
    each of the index's shape."""
    cols = [values] if isinstance(values, LweSampleArray) else list(values)
    if len(cols) != W or not all(isinstance(c, LweSampleArray) for c in cols):
        raise ValueError('a table of %d columns takes %d value arrays, got %d' % (W, W, len(cols)))
    if any(c.params != params.in_out_params for c in cols):
        raise ValueError('the values do not have the LWE parameters of this machine')
    if any(tuple(c.shape) != tuple(shape) for c in cols):
        raise ValueError('the values have shapes %s, the index %s' % ([tuple(c.shape) for c in cols], tuple(shape)))
    B, n = int(numpy.prod(shape, dtype=numpy.int64)), params.in_out_params.size
    a = torch.stack([c.a.reshape(B, n) for c in cols], 1)
    b = torch.stack([c.b.reshape(B) for c in cols], 1)
    var = torch.stack([c.current_variances.reshape(B).float() for c in cols]).amax(0) if B else torch.zeros(0)
    return a, b, [float(x) for x in var.cpu().numpy()]


def plain_values(thr, table, shape, W, values):
    """b (B, W) int32 of plain values broadcast to the index's shape: one array (or int) for every column, or a list of
    W.  'int' tables encode v 2^(31 - bits) mod 2^32 (so counts add up), 'bool' tables +-1/8."""
    cols = list(values) if isinstance(values, (list, tuple)) and len(values) == W and W > 1 else [values] * W
    B = int(numpy.prod(shape, dtype=numpy.int64))
    enc = []
    for c in cols:
        try:
            c = numpy.broadcast_to(numpy.asarray(c), shape)
        except ValueError:
            raise ValueError('values of shape %s do not broadcast to the index shape %s'
                             % (numpy.shape(c), tuple(shape))) from None
        if c.dtype.kind not in 'iub':
            raise ValueError('plain values must be integers, got %s' % c.dtype)
        if table.out == 'int':
            e = (c.astype(numpy.int64) << (31 - table.bits_out)) & 0xffffffff
        else:
            e = numpy.where(c != 0, int(MU), -int(MU)) & 0xffffffff
        enc.append(e.reshape(B).astype(numpy.uint32).view(numpy.int32))
    return thr.to_device(numpy.stack(enc, 1).reshape(B, W))


def scatter_passes(thr, params, keys, m, W, sels, a, b, accs, table_ids=None):
    """Add every query's value into its table: selector arrays `sels` (one per tenant, as lookup_passes), values a
    (B, W, n) under the cloud keys (None: plain values) and bodies b (B, W), the tables' int32 accumulators accs
    (T, P, 2, N) and, for T > 1, the table of each query (B,).  `keys` (OneKey, TenantKeys) serves the tree key switch."""
    k = params.tgsw_params.tlwe_params.mask_size
    for q0, q1, _, _, spec in selector_passes(thr, m, W, sels, table_ids is not None):
        Q = q1 - q0
        v = None
        if a is not None:
            v = keys.split(q0, q1).tree_keyswitch(a[q0:q1].reshape(Q * W, -1), k, per=W).reshape(Q, W, k + 1, N)
        delta = thr.index_write_assemble(v, b[q0:q1], m)
        del v
        ids = None if table_ids is None else table_ids[q0:q1]
        if m <= ROTATE_BITS:
            thr.index_write_rotate(delta, spec, m, accs, ids)
            continue
        cur = thr.index_write_rotate(delta, spec, m)
        del delta
        for j in range(m - 1, ROTATE_BITS, -1):
            cur = thr.index_demux_level(cur, spec, j)
        thr.index_demux_level(cur, spec, ROTATE_BITS, accs, ids)
        del cur


def finish(thr, params, table, acc, variance):
    """The EncryptedIndexTable of an accumulator: its 16-bit rounding, table's shape and encoding."""
    return EncryptedIndexTable(thr, params, table.bits, table.columns, _round16(acc), variance, table.out,
                               table.bits_out, table.single)


def differences(thr, table, shape, old, values):
    """The values v_q - old_q of a write, old the lookup of its indexes (one LweSampleArray per column), as
    LweSampleArrays (one per column), and the variances of the v_q: plain values count as trivial samples."""
    old = [old] if isinstance(old, LweSampleArray) else list(old)
    lwe_params = old[0].params
    W = table.columns
    B = int(numpy.prod(shape, dtype=numpy.int64))
    if isinstance(values, LweSampleArray) or (isinstance(values, (list, tuple)) and len(values) > 0
                                              and isinstance(values[0], LweSampleArray)):
        a, b, var = lwe_values(table.params, shape, W, values)
    else:
        b = plain_values(thr, table, shape, W, values)
        a, var = None, [0.0] * B
    out = []
    for w, o in enumerate(old):
        oa = o.a.reshape(B, -1).to(torch.int64)
        da = _wrap32(((0 if a is None else a[:, w].to(torch.int64)) - oa) & 0xffffffff)
        db = _wrap32((b[:, w].to(torch.int64) - o.b.reshape(B).to(torch.int64)) & 0xffffffff)
        out.append(LweSampleArray(lwe_params, da.reshape(tuple(shape) + (lwe_params.size,)), db.reshape(shape),
                                  o.current_variances.clone()))
    return out if W > 1 else out[0], var


def scatter_add(thr, params, tree_key, table, index, values, what='scatter_add', write_variances=None):
    """T[w, idx_q] += v_q[w] for every query (VirtualMachine.scatter_add); `write_variances` marks the values of a
    write (their per-query variances), whose noise rule differs."""
    lwe = check_arguments(what, params, index, table, tree_key, values)
    if table.out != 'int' and write_variances is None:
        raise ValueError("scatter_add adds integers: it takes out='int' tables only (write overwrites 'bool' entries)")
    m, W = table.bits, table.columns
    shape = index.shape
    B = int(numpy.prod(shape, dtype=numpy.int64))
    if lwe:
        a, b, var = lwe_values(params, shape, W, values)
    else:
        a, b, var = None, plain_values(thr, table, shape, W, values), None
    if write_variances is not None:
        var = write_variances
    variance = written_table_variance(params, leaf_variance(table), m, B, var, write_variances is not None)
    check_table_variance(params, variance, m, table.out, table.bits_out)
    acc = table_nodes(table)
    if B:
        scatter_passes(thr, params, OneKey(thr, tree_key=tree_key), m, W, [index.samples.reshape(B, m, 2, 2, 2, N)],
                       a, b, acc.reshape((1,) + tuple(acc.shape)))
    return finish(thr, params, table, acc, variance)


def write(thr, params, ks, tree_key, table, index, values):
    """T[idx_q] <- v_q (VirtualMachine.write): scatter_add of v_q - lookup(idx_q)."""
    check_arguments('write', params, index, table, tree_key, values)
    from .tree_lut import NuFHETreeKey
    if not isinstance(tree_key, NuFHETreeKey):
        raise TypeError('write needs a NuFHETreeKey (ctx.make_cloud_key(sk, tree_key=True)), got %s'
                        % type(tree_key).__name__)
    diffs, var = differences(thr, table, index.shape, lookup(thr, ks, index, table), values)
    return scatter_add(thr, params, tree_key, table, index, diffs, 'write', var)


def refresh_columns(thr, params, ks, table):
    """The entries of an encrypted table as LWE samples under the cloud key, (W, 2^m), ready for one bootstrap each:
    sample extraction of the 16-bit form (nb_compact_extract) and the key switch; a 'bool' entry's phase +-1/8 moved by
    +1/8 to the 1-bit integer encoding {0, 1/4}."""
    if not isinstance(table, EncryptedIndexTable):
        raise TypeError('refresh_table needs an EncryptedIndexTable, got %s' % type(table).__name__)
    if table.params != params:
        raise ValueError('the table was made for other parameters than this machine')
    rows = table.columns << table.bits
    a, b = thr.compact_extract(table.data, rows)
    ra, rb, _ = thr.keyswitch(ks.device_arrays(), (a, b))
    if table.out == 'bool':
        rb = _wrap32((rb.to(torch.int64) + int(MU)) & 0xffffffff)
    n = params.in_out_params.size
    shape = (table.columns, 1 << table.bits)
    cv = torch.full(shape, float(table.variance + keyswitch_variance(params)), dtype=torch.float32, device=rb.device)
    return LweSampleArray(params.in_out_params, ra.reshape(shape + (n,)), rb.reshape(shape), cv)


def refresh_table(vm, tree_key, table):
    """The same entries with fresh noise (VirtualMachine.refresh_table): W 2^m bootstraps of an identity vm.lut, then
    make_encrypted_table."""
    x = refresh_columns(vm.thread, vm.params, vm.cloud_key.keyswitch_key, table)
    if table.out == 'int':
        ident = vm.make_lut(numpy.arange(1 << table.bits_out), table.bits_out)
    else:
        ident = vm.make_lut(numpy.arange(2), 1, out='bool')
    y = vm.lut(ident, x)
    return make_encrypted_table(vm.thread, vm.params, tree_key, y[0] if table.single else y, table.out, table.bits_out)
