"""An independent NumPy restatement of the two new steps of tree-based programmable bootstrapping (DESIGN.md section
13): the LWE -> GLWE key switch and the test-vector assembly.  TEST INFRASTRUCTURE ONLY; it shares no code with the CUDA
source or nufhe_b200/tree_lut.py.

The key switch V (R, k+1, N) = D (R, n t) x T (n t, (k+1) N) is taken in float64 on the 16-bit halves of the key words
(every sum is below n t * 128 * 2^16 < 2^33, so exact), then recombined mod 2^32.  The assembly multiplies each G_m by
the polynomial W_m = X^(o_m) (1 + X + ... + X^(box - 1)) as a negacyclic matrix product, again on 16-bit halves."""
import numpy

import pack_ref
from pack_ref import N, u32, i32, digits, negacyclic_matrix


def keyswitch(a, masks, body):
    """V (R, k+1, N) int32 for LWE masks a (R, n) and the tree key's masks (n, t, k, N) and bodies (n, t, N)."""
    a = numpy.asarray(a)
    R = a.shape[0]
    K = pack_ref.key_polys(masks, body)                       # (n t, k+1, N)
    rows, k1, _ = K.shape
    Kw = u32(K).reshape(rows, k1 * N)
    lo, hi = (Kw & 0xffff).astype(numpy.float64), (Kw >> 16).astype(numpy.float64)
    d = digits(a).reshape(R, rows).astype(numpy.float64)
    return i32((d @ lo).astype(numpy.int64) + ((d @ hi).astype(numpy.int64) << 16)).reshape(R, k1, N)


def window(bits, m):
    """W_m = X^(o_m) Q_P as N integer coefficients (+-1 and 0)."""
    box = N >> bits
    w = numpy.zeros(N, numpy.int64)
    for e in range(m * box - box // 2, m * box + box - box // 2):
        e2 = e % (2 * N)
        if e2 < N:
            w[e2] += 1
        else:
            w[e2 - N] -= 1
    return w


def _mul(x, M):
    x = u32(x)
    return (x & 0xffff).astype(numpy.float64) @ M, (x >> 16).astype(numpy.float64) @ M


def assemble(v, b, bits):
    """tv (T, k+1, N) int32 from V (T, 2^bits, k+1, N) and the bodies b (T, 2^bits)."""
    v = numpy.asarray(v).astype(numpy.int64)
    b = numpy.asarray(b).astype(numpy.int64)
    T, M, k1, _ = v.shape
    G = -v
    G[:, :, k1 - 1, 0] += b
    tv = numpy.zeros((T, k1, N), numpy.int64)
    for m in range(M):
        W = negacyclic_matrix(window(bits, m))
        lo, hi = _mul(G[:, m].reshape(T * k1, N), W)
        tv = u32(tv + (lo.astype(numpy.int64) + (hi.astype(numpy.int64) << 16)).reshape(T, k1, N))
    return i32(tv)


def glwe_phase(tv, S):
    """Phase (T, N) of GLWE samples tv (T, k+1, N) under the binary key S (k, N)."""
    tv = numpy.asarray(tv)
    T, k1, _ = tv.shape
    acc = u32(tv[:, k1 - 1])
    for u in range(k1 - 1):
        lo, hi = _mul(tv[:, u], negacyclic_matrix(numpy.asarray(S)[u]))
        acc = u32(acc - lo.astype(numpy.int64) - (hi.astype(numpy.int64) << 16))
    return i32(acc)
