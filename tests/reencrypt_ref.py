"""An independent NumPy restatement of re-encryption (DESIGN.md section 22).  TEST INFRASTRUCTURE ONLY; it shares no
code with the CUDA source or nufhe_b200/reencrypt.py.

`reencrypt` takes the definition literally: (0, b) - sum_p d_p extract_p(C), with the extraction of every slot p of the
key's mask written out as a matrix (N, N) and the products taken in float64 on the 16-bit halves of the key words (every
sum is below n t 128 2^16 < 2^33, so exact).  `tree_chain` takes the other route the issue of this feature names: the
rotations X^(-p) C form a tree key (row i t + j encrypts the constant s_i g_j), whose key switch (tree_ref) gives V, and
the result is (0, b) minus the coefficient-0 extraction of V."""
import numpy

import tree_ref
from pack_ref import N, u32, i32, digits


def extraction_matrix(mask):
    """E (N, N): row p is the extracted mask of slot p of the polynomial `mask`, E[p, j] = mask[p - j] for j <= p and
    -mask[N + p - j] for j > p."""
    m = numpy.asarray(mask).astype(numpy.int64)
    p, j = numpy.meshgrid(numpy.arange(N), numpy.arange(N), indexing='ij')
    return numpy.where(j <= p, m[(p - j) % N], -m[(p - j) % N])


def _dot16(d, M):
    """d (R, K) small integers times M (K, N) int64, exact mod 2^32 through the 16-bit halves of M."""
    Mu = u32(M)
    lo, hi = (Mu & 0xffff).astype(numpy.float64), (Mu >> 16).astype(numpy.float64)
    df = d.astype(numpy.float64)
    return u32((df @ lo).astype(numpy.int64) + ((df @ hi).astype(numpy.int64) << 16))


def reencrypt(a, b, mask, body):
    """(out_a (R, N), out_b (R,)) int32 for LWE samples a (R, n), b (R,) and the key C = (mask (N,), body (N,))."""
    a = numpy.asarray(a).reshape(-1, numpy.asarray(a).shape[-1])
    R, n = a.shape
    d = digits(a).reshape(R, 2 * n)
    E = extraction_matrix(mask)[:2 * n]
    out_a = i32(-_dot16(d, E))
    bd = d.astype(numpy.int64) @ numpy.asarray(body).astype(numpy.int64)[:2 * n]
    out_b = i32(numpy.asarray(b).reshape(-1).astype(numpy.int64) - bd)
    return out_a, out_b


def rotate_down(P, p):
    """X^(-p) P (negacyclic): coefficient j is P[j + p] for j + p < N, else -P[j + p - N]."""
    P = numpy.asarray(P).astype(numpy.int64)
    j = numpy.arange(N)
    return numpy.where(j + p < N, P[(j + p) % N], -P[(j + p) % N])


def tree_key(mask, body, n):
    """The rotations X^(-p) C, p = i t + j, as a tree key: masks (n, 2, 1, N) and bodies (n, 2, N) int32."""
    masks = numpy.stack([i32(rotate_down(mask, p)) for p in range(2 * n)]).reshape(n, 2, 1, N)
    bodies = numpy.stack([i32(rotate_down(body, p)) for p in range(2 * n)]).reshape(n, 2, N)
    return masks, bodies


def from_tree_output(V, b):
    """(0, b) minus the coefficient-0 extraction of V (R, 2, N): out_a[0] = -V[0], out_a[j] = V[N - j], b - V_body[0]."""
    V = numpy.asarray(V).astype(numpy.int64)
    out_a = numpy.concatenate([-V[:, 0, :1], V[:, 0, :0:-1]], axis=1)
    return i32(out_a), i32(numpy.asarray(b).reshape(-1).astype(numpy.int64) - V[:, 1, 0])


def tree_chain(a, b, mask, body):
    a = numpy.asarray(a).reshape(-1, numpy.asarray(a).shape[-1])
    masks, bodies = tree_key(mask, body, a.shape[1])
    return from_tree_output(tree_ref.keyswitch(a, masks, bodies), b)


def phase(out_a, out_b, S):
    """Phase (R,) int32 of LWE samples under the extracted key of the GLWE key S (N,) binary: b - <a, S>."""
    s = numpy.asarray(S).astype(numpy.float64).reshape(-1)
    Au = u32(out_a)
    dot = u32((((Au & 0xffff).astype(numpy.float64) @ s).astype(numpy.int64))
              + (((Au >> 16).astype(numpy.float64) @ s).astype(numpy.int64) << 16))
    return i32(numpy.asarray(out_b).astype(numpy.int64) - dot)
