"""Oblivious writes composed from the oracle (TEST INFRASTRUCTURE): the delta assembly, the rotation by X^(+2^j) and
the demultiplexer levels of nufhe_b200/index_write.py, built from oracle.tgsw_external_mul with the rounded
decomposition (tests/index_ref.py), and the accumulation into the tables."""
import numpy

from oracle import oracle as O
import index_ref as R

N = 1024
ROTATE_BITS = 10


def assemble(v, b, m):
    """nb_index_write_assemble: v (Q, W, 2, N) int32 or None, b (Q, W) -> (Q, A, 2, N), (0, b_w) - V_w per column for
    m >= 10, sum_w X^(w 2^m) ((0, b_w) - V_w) below."""
    Q, W = b.shape
    d = numpy.zeros((Q, W, 2, N), numpy.int64)
    d[:, :, 1, 0] = b
    if v is not None:
        d -= v
    if m >= ROTATE_BITS:
        return (d & 0xffffffff).astype(numpy.uint32).view(numpy.int32)
    out = numpy.zeros((Q, 1, 2, N), numpy.int64)
    for w in range(W):
        sh = w << m
        out[:, 0, :, sh:] += d[:, w, :, :N - sh]
        out[:, 0, :, :sh] -= d[:, w, :, N - sh:]
    return (out & 0xffffffff).astype(numpy.uint32).view(numpy.int32)


def rotate(acc, sel_ref, rows):
    """acc (Q, A, 2, N); rows (Q, s): for j < s, ACC <- ACC + C_j [x] ((X^(+2^j) - 1) ACC)."""
    Q, A = acc.shape[:2]
    for j in range(rows.shape[1]):
        powers = numpy.full(Q * A, 1 << j, numpy.int32)
        tmp = O.shift_torus_polynomial(acc.reshape(Q * A, 2, N), powers, minus_one=True).reshape(acc.shape)
        acc = R.add(acc, R.apply(tmp, sel_ref, rows[:, j]))
    return acc


def demux_level(nodes, sel_ref, rows):
    """nodes (Q, K, 2, N) -> (Q, 2 K, 2, N): y -> (y - C [x] y, C [x] y), C = sel_ref[rows[q]]."""
    c = R.apply(nodes, sel_ref, rows)
    out = numpy.empty((nodes.shape[0], 2 * nodes.shape[1], 2, N), numpy.int32)
    out[:, 0::2] = R.sub(nodes, c)
    out[:, 1::2] = c
    return out


def accumulate(accs, leaves, table_ids):
    """accs (T, P, 2, N) + leaves (Q, P, 2, N) of query q into table table_ids[q], mod 2^32."""
    out = accs.astype(numpy.int64)
    for q in range(leaves.shape[0]):
        out[table_ids[q]] += leaves[q]
    return (out & 0xffffffff).astype(numpy.uint32).view(numpy.int32)


def leaves(delta, sel_ref, rows, m):
    """The leaves (Q, P, 2, N) of every query: the rotation of its deltas, then the demultiplexer for j = m-1 .. 10."""
    cur = rotate(delta, sel_ref, rows[:, :min(m, ROTATE_BITS)])
    for j in range(m - 1, ROTATE_BITS - 1, -1):
        cur = demux_level(cur, sel_ref, rows[:, j])
    return cur


def scatter(accs, delta, sel_ref, rows, m, table_ids=None):
    """The whole write into the accumulators accs (T, P, 2, N): delta (Q, A, 2, N) from assemble, sel_ref (R, 2, 2, 2,
    N), rows (Q, m) the row of selector j of query q."""
    ids = numpy.zeros(delta.shape[0], numpy.int64) if table_ids is None else numpy.asarray(table_ids)
    return accumulate(accs, leaves(delta, sel_ref, rows, m), ids)
