"""Encrypted-index lookups composed from the oracle (TEST INFRASTRUCTURE): CMux-tree levels and rotation steps built
from oracle.tgsw_external_mul, the exact NTT pinned to nufhe's, with selectors in the reference's transformed form
(oracle.bk_transform).  Layouts and steps as nufhe_b200/index_lookup.py describes them."""
import numpy

from oracle import oracle as O

N = 1024
ROTATE_BITS = 10
# The lookup kernels round the gadget decomposition where the oracle's (nufhe's) truncates: decomposing x + 2^11 with
# truncated digits is decomposing x with rounded ones, bit for bit.
ROUND = 1 << 11


def _u(x):
    return numpy.ascontiguousarray(x).view(numpy.uint32)


def add(x, y):
    return (_u(x) + _u(y)).view(numpy.int32)


def sub(x, y):
    return (_u(x) - _u(y)).view(numpy.int32)


def transform(rows):
    """Selector rows (..., 2, 2, 2, N) int32 -> (R, 2, 2, 2, N) uint64, the reference's form."""
    return O.bk_transform(numpy.ascontiguousarray(rows, numpy.int32).reshape(-1, 2, 2, 2, N))


def noiseless_selectors(bits_arr):
    """Trivial selectors b H: (..., m) bits -> (..., m, 2, 2, 2, N) int32, row (mi, j) = (0, .., b 2^(22 - 10 j) X^0
    on polynomial mi)."""
    bits_arr = numpy.asarray(bits_arr)
    out = numpy.zeros(bits_arr.shape + (2, 2, 2, N), numpy.int32)
    for mi in range(2):
        for j in range(2):
            out[..., mi, j, mi, 0] = bits_arr * (1 << (22 - 10 * j))
    return out


def table_polys(enc, m):
    """Encoded columns enc (W, 2^m) int32 -> the trivial samples (P, 2, N) int32 of the table's layout."""
    W = enc.shape[0]
    if m < ROTATE_BITS:
        plain = numpy.zeros((1, N), numpy.int32)
        plain[0, :W << m] = enc.reshape(-1)
    else:
        plain = enc.reshape(W << (m - ROTATE_BITS), N)
    polys = numpy.zeros((plain.shape[0], 2, N), numpy.int32)
    polys[:, 1] = plain
    return polys


def apply(x, sel_ref, rows):
    """x (Q, K, 2, N): sample k of query q times the selector row sel_ref[rows[q]] with the rounded decomposition, one
    oracle call per distinct row."""
    x = add(x, numpy.full(x.shape, ROUND, numpy.int32))
    out = numpy.empty_like(x)
    for r in numpy.unique(rows):
        qs = numpy.nonzero(rows == r)[0]
        out[qs] = O.tgsw_external_mul(x[qs].reshape(-1, 2, N), sel_ref, int(r)).reshape((len(qs),) + x.shape[1:])
    return out


def cmux_level(nodes, sel_ref, rows):
    """nodes (Q, 2 K, 2, N) -> (Q, K, 2, N): d_2i + C [x] (d_2i+1 - d_2i), C = sel_ref[rows[q]]."""
    d0, d1 = nodes[:, 0::2], nodes[:, 1::2]
    return add(d0, apply(sub(d1, d0), sel_ref, rows))


def rotate(acc, sel_ref, rows):
    """acc (Q, A, 2, N); rows (Q, s): for j < s, ACC <- ACC + C_j [x] ((X^(-2^j) - 1) ACC)."""
    Q, A = acc.shape[:2]
    for j in range(rows.shape[1]):
        powers = numpy.full(Q * A, 2 * N - (1 << j), numpy.int32)
        tmp = O.shift_torus_polynomial(acc.reshape(Q * A, 2, N), powers, minus_one=True).reshape(acc.shape)
        acc = add(acc, apply(tmp, sel_ref, rows[:, j]))
    return acc


def extract(acc, pos):
    """Sample extraction at coefficient pos of acc (..., 2, N): a (..., N), b (...)."""
    x = numpy.arange(N)
    A, B = acc[..., 0, :], acc[..., 1, :]
    a = numpy.where(x <= pos, A[..., (pos - x) % N], (0 - _u(A[..., (N + pos - x) % N])).view(numpy.int32))
    return a.astype(numpy.int32), B[..., pos].copy()


def rotate_extract(acc, sel_ref, rows, m, W):
    """nb_index_rotate_extract: acc (Q, A, 2, N) -> a (W, Q, N), b (W, Q)."""
    Q = acc.shape[0]
    acc = rotate(acc, sel_ref, rows[:, :min(m, ROTATE_BITS)])
    a = numpy.empty((W, Q, N), numpy.int32)
    b = numpy.empty((W, Q), numpy.int32)
    for w in range(W):
        if m >= ROTATE_BITS:
            a[w], b[w] = extract(acc[:, w], 0)
        else:
            a[w], b[w] = extract(acc[:, 0], w << m)
    return a, b


def lookup(polys, sel_ref, rows, m, W):
    """The whole lookup before the key switch: polys (P, 2, N) trivial table samples, sel_ref (R, 2, 2, 2, N), rows
    (Q, m) the row of sel_ref that is selector j of query q.  Returns a (W, Q, N), b (W, Q)."""
    Q = rows.shape[0]
    cur = numpy.broadcast_to(polys, (Q,) + polys.shape).copy()
    for j in range(ROTATE_BITS, m):
        cur = cmux_level(cur, sel_ref, rows[:, j])
    return rotate_extract(cur, sel_ref, rows, m, W)
