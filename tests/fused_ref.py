"""The fused bootstrap's entry points composed from the CPU oracle's steps (oracle/oracle.py): what every output of
nb_bootstrap_extract, nb_bootstrap_extract2, nb_bootstrap_lut_extract, nb_bootstrap_glwe_lut_extract, nb_blind_rotate
and nb_external_product is checked against.  TEST INFRASTRUCTURE ONLY; it shares no code with the CUDA source.

Every function takes host arrays and the same arguments as the engine method of the same name, with the key in the
reference's form (the first n rows of an OracleKeys.bk, or O.bk_transform of any integral key).  Any LWE dimension n
works; the prologue x = (0, c) + s1 x1 + s2 x2 wraps mod 2^32 as in the reference's lwe_affine.

The second part is shared by the GPU matrices: inputs whose first rows hit constructed edge values, outputs inside
guard rows, and the modes (one entry point with its inputs, the expected outputs and the C ABI call)."""
import types

import numpy
import torch

import gen_inputs as G
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

# ======== shared by the GPU matrices (tests/test_gpu_fused_matrix.py, tests/test_gpu_multibit_matrix.py) ============

STANDARD = types.SimpleNamespace(bootstrap_extract=bootstrap_extract, bootstrap_lut_extract=bootstrap_lut_extract,
                                 bootstrap_glwe_lut_extract=bootstrap_glwe_lut_extract)
GUARD = 3                                   # sentinel rows before and after every output
SENTINEL = 0x5A5A5A5A
EDGE_ROT = [0, 1, 1023, 1024, 1025, 2047]
TV_EDGES = [-2**31, 2**31 - 1, 0]


# ---- inputs with constructed edge rows ------------------------------------------------------------------------------

def _i32(v):
    v = int(v) % 2**32
    return v - 2**32 if v >= 2**31 else v


def _solve(target, s, rest):
    """x with s x = target - rest mod 2^32 (s = 2^k u, u odd; target - rest must be a multiple of 2^k)"""
    d = (int(target) - int(rest)) % 2**32
    k = ((s & -s).bit_length() - 1)
    assert d % (1 << k) == 0, (target, s, rest)
    return _i32((d >> k) * pow(s >> k, -1, 2**32))


def gate_targets():
    """prologue bodies / mask coefficients whose mod-switch to [0, 2N) is an edge value: the centre and the lower
    rounding tie of each"""
    return [v << 21 for v in EDGE_ROT] + [(v << 21) - 2**20 for v in EDGE_ROT]


def lut_targets(L):
    """the rounding ties of modswitch_lut: m 2^(21+L) + 2^(20+L) + {-1, 0, 1}, m = 0, 1, around N and at the wrap"""
    ms = [0, 1, 2**(10 - L) - 1, 2**(10 - L), 2**(11 - L) - 1]
    return [(m << (21 + L)) + (1 << (20 + L)) + d for m in ms for d in (-1, 0, 1)]


def cycled(T, B, n):
    """the targets of the first rows: row r takes T from position r on, cyclically, for its n mask coefficients and
    then its body"""
    return [[T[(r + i) % len(T)] for i in range(n + 1)] for r in range(min(B, len(T)))]


def paired(T, B, n):
    """the targets of the first rows for a multi-bit key (n even): every ordered pair (t, u) of T is the pair of mask
    coefficients (2g, 2g + 1) of one group g of one row, n / 2 pairs per row; the bodies cycle through T"""
    pairs = [(t, u) for t in T for u in T]
    G = n // 2
    rows = min(B, -(-len(pairs) // G))
    return [[v for g in range(G) for v in pairs[(r * G + g) % len(pairs)]] + [T[r % len(T)]] for r in range(rows)]


def lwe_inputs(rng, B, n, c, s1, s2, two, targets, even_only=False, layout=cycled):
    """x1 (and x2 if `two`) random, the first rows solved so that the prologue's body and mask coefficients take the
    values `targets` in the order `layout` gives: for x2 where s2 is odd, else for x1 with x2 = 0"""
    x1 = (G.torus32(rng, (B, n)), G.torus32(rng, (B,)))
    x2 = (G.torus32(rng, (B, n)), G.torus32(rng, (B,))) if two else None
    T = [t for t in targets if not even_only or t % 2 == 0]
    for r, row in enumerate(layout(T, B, n)):
        for i, t in enumerate(row):
            cc = int(c) if i == n else 0
            if two and s2 % 2:
                v1 = int(x1[1][r] if i == n else x1[0][r, i])
                v = _solve(t, s2, cc + s1 * v1)
                if i == n:
                    x2[1][r] = v
                else:
                    x2[0][r, i] = v
            else:
                if two:
                    if i == n:
                        x2[1][r] = 0
                    else:
                        x2[0][r, i] = 0
                v = _solve(t, s1, cc)
                if i == n:
                    x1[1][r] = v
                else:
                    x1[0][r, i] = v
    return x1, x2


def make_test_vectors(rng, rows, width=None):
    tv = G.torus32(rng, (rows, N) if width is None else (rows, width, N))
    flat = tv.reshape(-1, N)
    for r in range(min(flat.shape[0], 6)):
        flat[r, 0], flat[r, N - 1] = TV_EDGES[r % 3], TV_EDGES[(r + 1) % 3]
    return tv


# ---- modes: inputs, the oracle on rows `rows`, and the C ABI call ---------------------------------------------------
# `ref` holds the compositions the outputs are checked against (STANDARD: the ones above, for the standard key).

def ptr(t):
    return None if t is None else t.data_ptr()


def guarded(eng, rows, width):
    return torch.full((rows + 2 * GUARD, width), SENTINEL, dtype=torch.int32, device=eng.device)


def unguard(buf, what):
    h = buf.cpu().numpy()
    assert (h[:GUARD] == SENTINEL).all() and (h[-GUARD:] == SENTINEL).all(), 'a store outside the rows of ' + what
    return h[GUARD:-GUARD]


def to_dev(eng, x):
    return (None, None) if x is None else (eng.to_device(x[0]), eng.to_device(x[1]))


class Mode:
    """kind: gate, x2 (extract2, B = job batch), lut, glwe, explicit, plain.  want[k] holds output k for the
    ciphertexts (job rows for x2) `rows`, leading axis first; run() returns the same outputs for the batch's prefix."""

    def __init__(self, name, kind, n, want, rows, upload, call):
        self.name, self.kind, self.n, self.want, self.rows = name, kind, n, want, rows
        self.upload, self.call = upload, call
        self.key_free = False

    def check(self, got, B, what):
        k = int(numpy.searchsorted(self.rows, B))
        sel = self.rows[:k]
        for i, (g, w) in enumerate(zip(got, self.want)):
            assert (g[sel] == w[:k]).all(), (what, self.name, B, 'output', i)

    def equal(self, got, B):
        return self.row_equal(got, B)[1].all()

    def row_equal(self, got, B):
        """(the compared rows below B, whether every output of each equals the oracle)"""
        k = int(numpy.searchsorted(self.rows, B))
        sel = self.rows[:k]
        eq = numpy.ones(k, bool)
        for g, w in zip(got, self.want):
            eq &= (g[sel] == w[:k]).all(axis=tuple(range(1, g.ndim)))
        return sel, eq


def gate_mode(name, n, bk, c, s1, s2, mu, two, seed, B, rows=None, x=None, ref=STANDARD, layout=cycled):
    rng = G.rs(seed)
    x1, x2 = x if x is not None else lwe_inputs(rng, B, n, c, s1, s2, two, gate_targets(), even_only=s1 % 2 == 0,
                                                layout=layout)
    rows = numpy.arange(B) if rows is None else rows
    sub = lambda v: None if v is None else (v[0][rows], v[1][rows])   # noqa: E731
    want = ref.bootstrap_extract(sub(x1), sub(x2), c, s1, s2, mu, bk)

    def call(eng, dev, bk_int, b):
        (a1, b1), (a2, b2) = dev
        oa, ob = guarded(eng, b, N), guarded(eng, b, 1)
        eng._call('nb_bootstrap_extract', ptr(a1), ptr(b1), ptr(a2), ptr(b2), c, s1, s2, mu, bk_int.data_ptr(), n,
                  oa[GUARD].data_ptr(), ob[GUARD].data_ptr(), b)
        return unguard(oa, 'out_a'), unguard(ob, 'out_b')[:, 0]
    m = Mode(name, 'gate', n, want, rows, lambda eng: (to_dev(eng, x1), to_dev(eng, x2)), call)
    # mu = -2^31 is its own negation: the accumulator is the constant -2^31 at every step, whatever the key
    m.key_free = mu == -2**31
    return m


def x2_mode(name, n, bk, job_a, job_b, mu, seed, B, rows=None, ref=STANDARD, layout=cycled):
    """job = (c, s1, s2, two); every operand and constant of job B differs from job A's"""
    rng = G.rs(seed)
    xs = [lwe_inputs(rng, B, n, c, s1, s2, two, gate_targets(), even_only=s1 % 2 == 0, layout=layout)
          for c, s1, s2, two in (job_a, job_b)]
    rows = numpy.arange(B) if rows is None else rows
    sub = lambda v: None if v is None else (v[0][rows], v[1][rows])   # noqa: E731
    ja = (sub(xs[0][0]), sub(xs[0][1])) + tuple(job_a[:3])
    jb = (sub(xs[1][0]), sub(xs[1][1])) + tuple(job_b[:3])
    wa, wb = ref.bootstrap_extract(*ja, mu, bk), ref.bootstrap_extract(*jb, mu, bk)

    def call(eng, dev, bk_int, b):
        (a1, b1), (a2, b2), (c1, d1), (c2, d2) = dev
        oa, ob = guarded(eng, 2 * b, N), guarded(eng, 2 * b, 1)
        eng._call('nb_bootstrap_extract2', ptr(a1), ptr(b1), ptr(a2), ptr(b2), *job_a[:3],
                  ptr(c1), ptr(d1), ptr(c2), ptr(d2), *job_b[:3], mu, bk_int.data_ptr(), n,
                  oa[GUARD].data_ptr(), ob[GUARD].data_ptr(), b)
        ga, gb = unguard(oa, 'out_a'), unguard(ob, 'out_b')[:, 0]
        return ga[:b], gb[:b], ga[b:], gb[b:]
    return Mode(name, 'x2', n, (wa[0], wa[1], wb[0], wb[1]), rows,
                lambda eng: tuple(to_dev(eng, v) for v in (xs[0][0], xs[0][1], xs[1][0], xs[1][1])), call)


def lut_mode(name, n, bk, L, per_ct, two, seed, B, rows=None, ref=STANDARD, layout=cycled):
    rng = G.rs(seed)
    c, s1, s2 = (12345678, 2, -3) if two else (-987654, -1, 5)       # s2 is ignored without x2
    x1, x2 = lwe_inputs(rng, B, n, c, s1, s2, two, lut_targets(L), layout=layout)
    tv = make_test_vectors(rng, B if per_ct else 1)
    tv = tv if per_ct else tv[0]
    rows = numpy.arange(B) if rows is None else rows
    K = 1 << L
    sub = lambda v: None if v is None else (v[0][rows], v[1][rows])   # noqa: E731
    wa, wb = ref.bootstrap_lut_extract(sub(x1), sub(x2), c, s1, s2, tv[rows] if per_ct else tv, L, bk)

    def call(eng, dev, bk_int, b):
        (a1, b1), (a2, b2), dtv = dev
        oa, ob = guarded(eng, b * K, N), guarded(eng, b * K, 1)
        eng._call('nb_bootstrap_lut_extract', ptr(a1), ptr(b1), ptr(a2), ptr(b2), c, s1, s2, dtv.data_ptr(),
                  N if per_ct else 0, L, bk_int.data_ptr(), n, oa[GUARD].data_ptr(), ob[GUARD].data_ptr(), b)
        return unguard(oa, 'out_a').reshape(b, K, N), unguard(ob, 'out_b').reshape(b, K)
    return Mode(name, 'lut', n, (wa.reshape(-1, K, N), wb.reshape(-1, K)), rows,
                lambda eng: (to_dev(eng, x1), to_dev(eng, x2), eng.to_device(tv)), call)


def glwe_mode(name, n, bk, seed, B, rows=None, ref=STANDARD, layout=cycled, tv=None):
    """tv: the test vectors (B, 2, N), random with edge coefficients if None"""
    rng = G.rs(seed)
    x, _ = lwe_inputs(rng, B, n, 0, 1, 0, False, gate_targets() + lut_targets(0), layout=layout)
    tv = make_test_vectors(rng, B, 2) if tv is None else tv
    rows = numpy.arange(B) if rows is None else rows
    want = ref.bootstrap_glwe_lut_extract((x[0][rows], x[1][rows]), tv[rows], bk)

    def call(eng, dev, bk_int, b):
        (a, bb), dtv = dev
        oa, ob = guarded(eng, b, N), guarded(eng, b, 1)
        eng._call('nb_bootstrap_glwe_lut_extract', ptr(a), ptr(bb), dtv.data_ptr(), bk_int.data_ptr(), n,
                  oa[GUARD].data_ptr(), ob[GUARD].data_ptr(), b)
        return unguard(oa, 'out_a'), unguard(ob, 'out_b')[:, 0]
    return Mode(name, 'glwe', n, want, rows, lambda eng: (to_dev(eng, x), eng.to_device(tv)), call)
