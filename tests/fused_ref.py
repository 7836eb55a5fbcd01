"""The fused bootstrap's entry points composed from the CPU oracle's steps (oracle/oracle.py): what every output of
nb_bootstrap_extract, nb_bootstrap_extract2, nb_bootstrap_lut_extract, nb_bootstrap_glwe_lut_extract, nb_blind_rotate
and nb_external_product is checked against.  TEST INFRASTRUCTURE ONLY; it shares no code with the CUDA source.

Every function takes host arrays and the same arguments as the engine method of the same name, with the key in the
reference's form (the first n rows of an OracleKeys.bk, or O.bk_transform of any integral key).  Any LWE dimension n
works; the prologue x = (0, c) + s1 x1 + s2 x2 wraps mod 2^32 as in the reference's lwe_affine."""
import numpy

from oracle import oracle as O

N = 1024


def i32(x):
    return (numpy.asarray(x).astype(numpy.int64) & 0xffffffff).astype(numpy.uint32).view(numpy.int32)


def prologue(x1, x2, c, s1, s2):
    """(a, b) of (0, c) + s1 x1 + s2 x2; x2 may be None"""
    a = numpy.asarray(x1[0]).astype(numpy.int64) * s1
    b = numpy.asarray(x1[1]).astype(numpy.int64) * s1 + c
    if x2 is not None:
        a = a + numpy.asarray(x2[0]).astype(numpy.int64) * s2
        b = b + numpy.asarray(x2[1]).astype(numpy.int64) * s2
    return i32(a), i32(b)


def bootstrap_extract(x1, x2, c, s1, s2, mu, bk):
    """The gate bootstrap without key switch: the extracted sample (a (B, N), b (B,))."""
    a, b = prologue(x1, x2, c, s1, s2)
    return O.bootstrap(a, b, bk[:a.shape[-1]], None, mu)


def bootstrap_extract2(job_a, job_b, mu, bk):
    """Two independent gates, job = (x1, x2, c, s1, s2); rows of job B follow those of job A."""
    ra = bootstrap_extract(*job_a, mu, bk)
    rb = bootstrap_extract(*job_b, mu, bk)
    return numpy.concatenate([ra[0], rb[0]]), numpy.concatenate([ra[1], rb[1]])


def _extract_outputs(acc, L):
    """samples j = 0 .. 2^L - 1 of every accumulator: a rotation by X^(2N - j), then the extraction; rows c 2^L + j"""
    B, K = acc.shape[0], 1 << L
    out_a, out_b = numpy.empty((B, K, N), numpy.int32), numpy.empty((B, K), numpy.int32)
    for j in range(K):
        src = O.shift_torus_polynomial(acc, numpy.full(B, 2 * N - j, numpy.int32)) if j else acc
        out_a[:, j], out_b[:, j] = O.tlwe_extract_lwe_samples(src)
    return out_a.reshape(B * K, N), out_b.reshape(B * K)


def oracle_lut(a, b, tv, L, bk):
    """The reference's composition for x = (a, b): t32_to_phase (2N / 2^L) * 2^L, X^(2N - barb) * tv, trivial
    accumulator, blind rotation, then per output j a rotation by X^(2N - j) and the extraction; rows c * 2^L + j."""
    B = b.size
    barb = (O.t32_to_phase(b, (2 * N) >> L).astype(numpy.int64) << L).astype(numpy.int32)
    bara = (O.t32_to_phase(a, (2 * N) >> L).astype(numpy.int64) << L).astype(numpy.int32)
    tvs = numpy.ascontiguousarray(numpy.broadcast_to(tv.reshape(-1, N), (B, N)))
    acc = O.tlwe_noiseless_trivial(O.shift_torus_polynomial(tvs[:, None, :], barb, invert_powers=True)[:, 0])
    acc = O.blind_rotate(acc, bk[:a.shape[-1]], bara)
    return _extract_outputs(acc, L)


def bootstrap_lut_extract(x1, x2, c, s1, s2, tv, L, bk):
    """The programmable bootstrap: tv (N,) shared by the batch or (B, N) one per ciphertext."""
    a, b = prologue(x1, x2, c, s1, s2)
    return oracle_lut(a, b, numpy.asarray(tv), L, bk)


def bootstrap_glwe_lut_extract(x, tv, bk):
    """The programmable bootstrap with one GLWE test vector (mask, body) per ciphertext, tv (B, 2, N): both
    polynomials times X^(2N - barb), blind rotation, extraction."""
    a, b = i32(x[0]), i32(x[1])
    barb = O.t32_to_phase(b, 2 * N)
    bara = O.t32_to_phase(a, 2 * N)
    acc = O.shift_torus_polynomial(numpy.asarray(tv, numpy.int32), barb, invert_powers=True)
    acc = O.blind_rotate(acc, bk[:a.shape[-1]], bara)
    return O.tlwe_extract_lwe_samples(acc)


def blind_rotate(accum, bara, bk):
    """The explicit blind rotation: (out_a, out_b, accum_out)."""
    acc = O.blind_rotate(accum, bk[:bara.shape[-1]], bara)
    out_a, out_b = O.tlwe_extract_lwe_samples(acc)
    return out_a, out_b, acc


def external_product(accum, bk, row):
    """One plain external product bk[row] (x) accum."""
    return O.tgsw_external_mul(accum, bk, row)
