"""An independent NumPy restatement of public-key encryption (DESIGN.md section 11): the reference nb_pk_encrypt and
its host emulation are checked against.  TEST INFRASTRUCTURE ONLY; it shares no code with the CUDA source.

    a_c = sum_i r_ci A_i,  b_c = mu_c + sum_i r_ci b_i  (mod 2^32),  cv_c = float32(popcount(r_c)) * float32(variance)

with bit i of R's row c = bit i % 32 of word (c, i // 32).  The product is taken in float64: every partial sum is below
m * 2^32 <= 2^46, so it is exact whatever the summation order, and reduced mod 2^32 afterwards."""
import numpy

from chacha_ref import seeded_uniform


def r_bits(r_words, m):
    """(B, m) 0/1 float64 matrix R from its (B, m/32) words."""
    w = numpy.asarray(r_words).astype(numpy.int64).astype(numpy.uint32).reshape(-1, m // 32)
    bits = (w[:, :, None] >> numpy.arange(32, dtype=numpy.uint32)) & 1
    return bits.reshape(w.shape[0], m).astype(numpy.float64)


def _mod32(x):
    return (numpy.fmod(x, 2.0**32).astype(numpy.int64) & 0xffffffff).astype(numpy.uint32).view(numpy.int32)


def encrypt(masks, pk_b, r_words, mus, variance, rows_per_step=256):
    """(a (B, n), b (B,), cv (B,)) for masks A (m, n), bodies b (m,), R words (B, m/32) and messages (B,)."""
    masks = numpy.asarray(masks)
    m, n = masks.shape
    W = numpy.empty((m, n + 1), numpy.float64)
    W[:, :n] = masks.astype(numpy.int64) & 0xffffffff
    W[:, n] = numpy.asarray(pk_b).astype(numpy.int64) & 0xffffffff
    r_words = numpy.asarray(r_words).reshape(-1, m // 32)
    B = r_words.shape[0]
    a, b = numpy.empty((B, n), numpy.int32), numpy.empty(B, numpy.int32)
    pop = numpy.empty(B, numpy.float64)
    for c0 in range(0, B, rows_per_step):
        R = r_bits(r_words[c0:c0 + rows_per_step], m)
        P = R @ W
        a[c0:c0 + len(R)] = _mod32(P[:, :n])
        b[c0:c0 + len(R)] = _mod32(P[:, n] + (numpy.asarray(mus).reshape(-1)[c0:c0 + len(R)].astype(numpy.int64) & 0xffffffff))
        pop[c0:c0 + len(R)] = R.sum(1)
    cv = pop.astype(numpy.float32) * numpy.float32(variance)
    return a, b, cv


def encrypt_with_seed(pk_seed, pk_b, n, r_words, mus, variance):
    """The same with the masks regenerated from the public key's seed (stream (seed, nonce 0), shape (m, n))."""
    return encrypt(seeded_uniform(pk_seed, 0, (len(pk_b), n)), pk_b, r_words, mus, variance)


def planes(masks, pk_b):
    """nb_pk_prepare's output: byte p of W[k][col], W = [A | b | 1 | 0...] padded to a multiple of 8 columns, at
    ((p * npad + col) * m + k)."""
    masks = numpy.asarray(masks)
    m, n = masks.shape
    npad = (n + 2 + 7) // 8 * 8
    W = numpy.zeros((m, npad), numpy.uint32)
    W[:, :n] = masks.astype(numpy.int64) & 0xffffffff
    W[:, n] = numpy.asarray(pk_b).astype(numpy.int64) & 0xffffffff
    W[:, n + 1] = 1
    return numpy.ascontiguousarray(W.view(numpy.uint8).reshape(m, npad, 4).transpose(2, 1, 0)).reshape(-1)
