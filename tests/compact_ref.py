"""An independent NumPy restatement of compact public-key encryption (DESIGN.md section 16) without the NTT: what
nb_compact_finish, nb_compact_extract, ctx.encrypt with a compact key and vm.expand are checked against.  TEST
INFRASTRUCTURE ONLY; it shares no code with the CUDA source or nufhe_b200/compact.py.

The negacyclic products A_u r are taken in int64 as x @ M(r), M(r) the (N, N) matrix of multiplication by r: with r
binary every coefficient is a sum of at most N int32 values, below 2^41.  Extraction is written out from its formula,
and the key switch is the oracle's."""
import numpy

from oracle import oracle as O

N = 1024


def u32(x):
    return numpy.asarray(x).astype(numpy.int64) & 0xffffffff


def i32(x):
    return u32(x).astype(numpy.uint32).view(numpy.int32)


def round16(x):
    return ((u32(x) + 2**15) >> 16 & 0xffff).astype(numpy.uint16)


def unround16(v):
    return i32(numpy.asarray(v).astype(numpy.int64) << 16)


def r_bits(words):
    """(G, N) binary polynomials from the words (G, N / 32): bit i of group g = bit i % 32 of word (g, i // 32)."""
    w = u32(words)
    return ((w[:, :, None] >> numpy.arange(32)[None, None, :]) & 1).reshape(w.shape[0], N)


def negacyclic_matrix(s):
    """M (N, N) int64 with (x * s) = x @ M for the negacyclic product by the polynomial s."""
    s = numpy.asarray(s).astype(numpy.int64)
    x = numpy.arange(N)[:, None]
    y = numpy.arange(N)[None, :]
    return s[(y - x) % N] * numpy.where(y >= x, 1, -1)


def products(polys, r):
    """(G, k+1, N) int64 in [0, 2^32): the key polynomials (k+1, N) times each group's r (G, N), negacyclic."""
    polys = numpy.asarray(polys).astype(numpy.int64)
    return numpy.stack([u32(polys @ negacyclic_matrix(rg)) for rg in numpy.asarray(r)])


def finish(C, e1, e2, mus):
    """The uint16 data (G, k+1, N) from the products C, noises e1 (G, k, N), e2 (G, N) and messages mus (B,)."""
    C = numpy.asarray(C).astype(numpy.int64)
    G, k1, _ = C.shape
    mus = numpy.asarray(mus).reshape(-1).astype(numpy.int64)
    v = C.copy()
    v[:, :k1 - 1] += numpy.asarray(e1).astype(numpy.int64)
    body = numpy.zeros(G * N, numpy.int64)
    body[:mus.size] = mus
    v[:, k1 - 1] += numpy.asarray(e2).astype(numpy.int64) + body.reshape(G, N)
    out = round16(v)
    occupied = numpy.arange(G * N).reshape(G, N) < mus.size
    out[:, k1 - 1][~occupied] = 0
    return out


def encrypt(polys, words, e1, e2, mus):
    return finish(products(polys, r_bits(words)), e1, e2, mus)


def extract(data, rows):
    """The extracted samples a (rows, k N), b (rows,) int32 of the first `rows` slots of data (G, k+1, N)."""
    x = unround16(data).astype(numpy.int64)                              # (G, k+1, N)
    G, k1, _ = x.shape
    k = k1 - 1
    a = numpy.empty((rows, k * N), numpy.int64)
    b = numpy.empty(rows, numpy.int64)
    j = numpy.arange(N)
    for c in range(rows):
        g, p = divmod(c, N)
        for u in range(k):
            A = x[g, u]
            a[c, u * N:(u + 1) * N] = numpy.where(j <= p, A[(p - j) % N], -A[(N + p - j) % N])
        b[c] = x[g, k, p]
    return i32(a), i32(b)


def keyswitch(ks, a, b):
    """The cloud key's key switch (the oracle's), ks = (ks_a, ks_b, ks_cv) host arrays: (a, b, cv)."""
    return O.lwe_keyswitch(ks[0], ks[1], ks[2], a, b)


def expand(data, rows, ks):
    return keyswitch(ks, *extract(data, rows))


def phases(data, S):
    """Torus32 phases (G N,) of compact data under the binary key S (k, N): coefficient p of body' - sum_u A'_u S_u."""
    x = unround16(data).astype(numpy.int64)
    G, k1, _ = x.shape
    acc = x[:, k1 - 1].copy()
    for u in range(k1 - 1):
        acc -= x[:, u] @ negacyclic_matrix(numpy.asarray(S)[u])
    return i32(acc).reshape(-1)


def noise_terms(params):
    """(fresh, mask rounding, body rounding, key switch) variances of an expanded sample, k = params' mask size:
    E r + e2 - e1 S with r and S binary of weight about N / 2 per polynomial, the 16-bit rounding of the k N masks, each
    meeting a key bit half the time, and of the body, and t digits of base 4 per extracted coefficient, 3/4 of them
    non-zero, each adding one key-switch-key row's variance."""
    tl = params.tgsw_params.tlwe_params
    k = tl.mask_size
    sigma2 = tl.min_noise**2
    q = 2.0**-32 / 12
    ks = k * N * params.ks_decomp_length * 0.75 * params.in_out_params.min_noise**2
    return (N / 2 + k * N / 2 + 1) * sigma2, k * N / 2 * q, q, ks
