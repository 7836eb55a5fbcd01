"""An independent NumPy restatement of result packing (DESIGN.md section 12) without the NTT: what nb_pack_digits,
nb_ntt_mac, nb_pack_finish and vm.pack are checked against.  TEST INFRASTRUCTURE ONLY; it shares no code with the CUDA
source or nufhe_b200/packing.py.

For input c (group g = c // N, slot p = c % N) the polynomial sum_ij d_cij K_ij is one row of a matrix product: the
digits d (B, n t) times the key K (n t, (k+1) N).  It is taken in float64 on the 16-bit halves of the key words, where
every sum is below n t * 128 * 2^16 < 2^33 and so exact, then recombined mod 2^32 in int64, multiplied by X^p (a
negacyclic rotation) and summed per group."""
import numpy

N = 1024
GADGET = (2**24, 2**16)


def u32(x):
    return numpy.asarray(x).astype(numpy.int64) & 0xffffffff


def i32(x):
    return u32(x).astype(numpy.uint32).view(numpy.int32)


def digits(a):
    """(..., t = 2) digits of the mask words a: w = a + 2^15 + 2^23 + 2^31, d0 = (w >> 24) - 128,
    d1 = ((w >> 16) & 255) - 128."""
    w = u32(numpy.asarray(a).astype(numpy.int64) + 2**15 + 2**23 + 2**31)
    return numpy.stack([(w >> 24) - 128, ((w >> 16) & 255) - 128], -1)


def round16(x):
    return ((u32(x) + 2**15) >> 16 & 0xffff).astype(numpy.uint16)


def unround16(v):
    return i32(numpy.asarray(v).astype(numpy.int64) << 16)


def rotate(P, p):
    """X^p * P for polynomials P (M, ..., N) and powers p (M,) in [0, N), negacyclic, int64."""
    y = numpy.arange(N)
    idx = (y[None, :] - p[:, None]) % N                                      # (M, N)
    sign = numpy.where(y[None, :] < p[:, None], -1, 1)
    idx = idx.reshape((P.shape[0],) + (1,) * (P.ndim - 2) + (N,))
    sign = sign.reshape(idx.shape)
    return numpy.take_along_axis(P, numpy.broadcast_to(idx, P.shape), -1) * sign


def key_polys(masks, body):
    """K (n t, k+1, N) from the masks (n, t, k, N) and bodies (n, t, N)."""
    masks, body = numpy.asarray(masks), numpy.asarray(body)
    n, t, k, _ = masks.shape
    return numpy.concatenate([masks, body[:, :, None, :]], axis=2).reshape(n * t, k + 1, N)


def pack_products(a, K):
    """C (G, k+1, N) int64 in [0, 2^32): C_g = sum_{c in g} X^p sum_ij d_cij K_ij."""
    a = numpy.asarray(a).reshape(-1, numpy.asarray(a).shape[-1])
    B = a.shape[0]
    R, k1, _ = K.shape
    Kw = u32(K).reshape(R, k1 * N)
    lo, hi = (Kw & 0xffff).astype(numpy.float64), (Kw >> 16).astype(numpy.float64)
    G = -(-B // N)
    C = numpy.zeros((G, k1, N), numpy.int64)
    for g in range(G):
        c0, c1 = g * N, min(B, (g + 1) * N)
        d = digits(a[c0:c1]).reshape(c1 - c0, R).astype(numpy.float64)
        P = (u32((d @ lo).astype(numpy.int64) + ((d @ hi).astype(numpy.int64) << 16))).reshape(c1 - c0, k1, N)
        C[g] = u32(rotate(P, numpy.arange(c1 - c0)).sum(0))
    return C


def finish(C, b):
    """The uint16 output (G, k+1, N) from C and the bodies b (B,)."""
    G, k1, _ = C.shape
    bodies = numpy.zeros(G * N, numpy.int64)
    b = numpy.asarray(b).reshape(-1).astype(numpy.int64)
    bodies[:b.size] = b
    v = -C
    v[:, k1 - 1] += bodies.reshape(G, N)
    return round16(v)


def pack(a, b, K):
    """The packed data (G, k+1, N) uint16 of LWE samples a (B, n), b (B,) with key polynomials K (n t, k+1, N)."""
    return finish(pack_products(a, K), b)


def noise_terms(params, slots=N):
    """Variances (torus units) that packing adds to a phase, for a group of `slots` inputs with uniform masks:
    the packing-key noise n t slots E[d^2] sigma^2 (every slot collects the key noise of all slots' digits), the rounding
    of the masks before the decomposition (n / 2) 2^-32 / 12, and the 16-bit mod switch of the output
    (k N / 2 + 1) 2^-32 / 12."""
    n = params.in_out_params.size
    tl = params.tgsw_params.tlwe_params
    d2 = ((256**2 - 1) / 12 + 0.25)                     # E[d^2], d uniform in [-128, 127]
    key = n * len(GADGET) * slots * d2 * tl.min_noise**2
    rnd = n / 2 * 2.0**-32 / 12
    ms = (tl.mask_size * tl.polynomial_degree / 2 + 1) * 2.0**-32 / 12
    return key, rnd, ms


def negacyclic_matrix(s):
    """M (N, N) with (x * s) = x @ M for the negacyclic product by the polynomial s."""
    s = numpy.asarray(s).astype(numpy.int64)
    x = numpy.arange(N)[:, None]
    y = numpy.arange(N)[None, :]
    return (s[(y - x) % N] * numpy.where(y >= x, 1, -1)).astype(numpy.float64)


def phases(data, S):
    """Torus32 phases (G * N,) of packed data (G, k+1, N) under the binary key S (k, N): unround, then
    body - sum_u mask_u * S_u, every product exact on 16-bit halves in float64."""
    data = numpy.asarray(data)
    G, k1, _ = data.shape
    x = u32(unround16(data))
    acc = u32(x[:, k1 - 1])
    for u in range(k1 - 1):
        M = negacyclic_matrix(numpy.asarray(S)[u])
        lo, hi = (x[:, u] & 0xffff).astype(numpy.float64), (x[:, u] >> 16).astype(numpy.float64)
        prod = (lo @ M).astype(numpy.int64) + ((hi @ M).astype(numpy.int64) << 16)
        acc = u32(acc - prod)
    return i32(acc).reshape(-1)
