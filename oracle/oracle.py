"""ctypes front end of oracle/nufhe_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Only tests/, __graft_entry__.smoke() and the cpu_baseline / --impl reference legs of bench.py may import
this module.  Every function takes and returns host NumPy arrays with the reference's layouts
(SURVEY.md Appendix C).  Reference citations are in the C source next to each restated function.

Key generation here follows the reference's host-side RNG draw order (SURVEY.md Appendix E) so that a
seed reproduces nufhe's keys bit for bit:
  nufhe/api_low_level.py:242-250, lwe.py:77-79, tlwe.py:83-92, bootstrap.py:59-76, tlwe.py:184-197,
  tlwe_cpu.py:64-89, tgsw_cpu.py:109-126, tlwe_gpu.py:199-236, lwe.py:265-295, lwe_cpu.py:26-59.
"""
import ctypes
import os
import subprocess

import numpy

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, 'libnufhe_oracle.so')

N = 1024          # nufhe/api_low_level.py:49
LWE_N = 500       # :50
KS_T = 8          # :55
KS_LOG2_BASE = 2  # :56
P = 2**64 - 2**32 + 1
_COEFF = (2 / numpy.pi) ** 0.5
KS_STDEV = 1 / 2**15 * _COEFF      # api_low_level.py:58
BS_STDEV = 9e-9 * _COEFF           # :59
MU = numpy.int32(2**29)            # phase_to_t32(1, 8), numeric_functions.py:30-31


def build(force=False):
    """(Re)compile libnufhe_oracle.so when it is missing or older than nufhe_oracle.c."""
    src = os.path.join(_HERE, 'nufhe_oracle.c')
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(src):
        subprocess.check_call(['make', '-C', _HERE, '-s', 'libnufhe_oracle.so'])
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = ctypes.CDLL(_LIB_PATH)
        _lib.orc_selftest.restype = ctypes.c_int
        _lib.orc_selftest.argtypes = [ctypes.c_uint64, ctypes.c_size_t]
        _lib.orc_init()
    return _lib


def set_threads(n):
    """Number of OpenMP threads the C oracle uses (bench.py sets it to the usable host cores)."""
    lib().orc_set_threads(ctypes.c_int(int(n)))


def get_threads():
    return int(lib().orc_get_threads())


def _p(arr):
    return arr.ctypes.data_as(ctypes.c_void_p)


def _c(arr, dtype):
    return numpy.ascontiguousarray(arr, dtype=dtype)


_sz = ctypes.c_size_t


def selftest(seed=1, n=100000):
    return lib().orc_selftest(seed, n)


# ---------------------------------------------------------------- field ops

def _ff_binary(name, a, b):
    a = _c(a, numpy.uint64)
    b = _c(numpy.broadcast_to(b, a.shape), numpy.uint64)
    out = numpy.empty_like(a)
    getattr(lib(), name)(_p(out), _p(a), _p(b), _sz(a.size))
    return out


def ff_mul(a, b): return _ff_binary('orc_ff_mul', a, b)
def ff_add(a, b): return _ff_binary('orc_ff_add', a, b)
def ff_sub(a, b): return _ff_binary('orc_ff_sub', a, b)
def ff_mul_prepared(a, b): return _ff_binary('orc_ff_mul_prepared', a, b)


def ff_prepare_for_mul(a):
    a = _c(a, numpy.uint64)
    out = numpy.empty_like(a)
    lib().orc_ff_prepare_for_mul(_p(out), _p(a), _sz(a.size))
    return out


def ff_lsh(a, s):
    a = _c(a, numpy.uint64)
    s = _c(numpy.broadcast_to(s, a.shape), numpy.uint32)
    out = numpy.empty_like(a)
    lib().orc_ff_lsh(_p(out), _p(a), _p(s), _sz(a.size))
    return out


# ---------------------------------------------------------------- transforms

def _batch(arr):
    assert arr.shape[-1] == N
    return arr.size // N


def ntt_forward_i32(x):
    x = _c(x, numpy.int32)
    out = numpy.empty(x.shape, numpy.uint64)
    lib().orc_ntt_forward_i32(_p(out), _p(x), _sz(_batch(x)))
    return out


def ntt_forward_u64(x):
    x = _c(x, numpy.uint64)
    out = numpy.empty(x.shape, numpy.uint64)
    lib().orc_ntt_forward_u64(_p(out), _p(x), _sz(_batch(x)))
    return out


def ntt_inverse_u64(x):
    x = _c(x, numpy.uint64)
    out = numpy.empty(x.shape, numpy.uint64)
    lib().orc_ntt_inverse_u64(_p(out), _p(x), _sz(_batch(x)))
    return out


def ntt_inverse_i32(x):
    x = _c(x, numpy.uint64)
    out = numpy.empty(x.shape, numpy.int32)
    lib().orc_ntt_inverse_i32(_p(out), _p(x), _sz(_batch(x)))
    return out


# ---------------------------------------------------------------- scheme pieces

def t32_to_phase(x, mspace_size):
    x = _c(x, numpy.int32)
    out = numpy.empty_like(x)
    lib().orc_t32_to_phase(_p(out), _p(x), _sz(x.size), ctypes.c_uint32(mspace_size))
    return out


def shift_torus_polynomial(source, powers, powers_idx=None, minus_one=False, invert_powers=False):
    """source (B, polys, N); powers (B,) or (B, n) with powers_idx."""
    source = _c(source, numpy.int32)
    powers = _c(powers, numpy.int32)
    B = source.shape[0]
    polys = source.size // (B * N)
    if powers_idx is None:
        stride, idx = 1, 0
        assert powers.size == B
    else:
        stride, idx = powers.shape[-1], powers_idx
    out = numpy.empty_like(source)
    lib().orc_shift_torus_polynomial(
        _p(out), _p(source), _p(powers), _sz(B), _sz(polys), _sz(stride), _sz(idx),
        ctypes.c_int(int(minus_one)), ctypes.c_int(int(invert_powers)))
    return out


def tlwe_noiseless_trivial(mu):
    mu = _c(mu, numpy.int32)
    B = mu.size // N
    acc = numpy.empty((B, 2, N), numpy.int32)
    lib().orc_tlwe_noiseless_trivial(_p(acc), _p(mu), _sz(B))
    return acc


def tlwe_extract_lwe_samples(acc):
    acc = _c(acc, numpy.int32)
    B = acc.size // (2 * N)
    a = numpy.empty((B, N), numpy.int32)
    b = numpy.empty((B,), numpy.int32)
    lib().orc_tlwe_extract_lwe_samples(_p(a), _p(b), _p(acc), _sz(B))
    return a, b


def tgsw_decompose(sample):
    sample = _c(sample, numpy.int32)
    B = sample.size // (2 * N)
    out = numpy.empty((B, 2, 2, N), numpy.int32)
    lib().orc_tgsw_decompose(_p(out), _p(sample), _sz(B))
    return out


def tgsw_mac(tr, bk, bk_row):
    tr = _c(tr, numpy.uint64)
    bk = _c(bk, numpy.uint64)
    B = tr.size // (4 * N)
    out = numpy.empty((B, 2, N), numpy.uint64)
    lib().orc_tgsw_mac(_p(out), _p(tr), _p(bk), _sz(bk_row), _sz(B))
    return out


def tgsw_external_mul(accum, bk, bk_row):
    """Returns bk[bk_row] (x) accum (the reference overwrites accum in place)."""
    out = _c(accum, numpy.int32).copy()
    bk = _c(bk, numpy.uint64)
    lib().orc_tgsw_external_mul(_p(out), _p(bk), _sz(bk_row), _sz(out.size // (2 * N)))
    return out


def tgsw_decompose_k(sample):
    """Gadget decomposition of (..., N) polynomials -> (..., 2, N), any number of polynomials per sample."""
    sample = _c(sample, numpy.int32)
    out = numpy.empty(sample.shape[:-1] + (2, N), numpy.int32)
    lib().orc_tgsw_decompose_polys(_p(out), _p(sample), _sz(sample.size // N))
    return out


def tgsw_mac_k(tr, bk_row):
    """tr (B, k+1, 2, N), bk_row (k+1, 2, k+1, N) -> (B, k+1, N), any mask size k."""
    tr = _c(tr, numpy.uint64)
    bk_row = _c(bk_row, numpy.uint64)
    k1 = bk_row.shape[0]
    B = tr.size // (k1 * 2 * N)
    out = numpy.empty((B, k1, N), numpy.uint64)
    lib().orc_tgsw_mac_k(_p(out), _p(tr), _p(bk_row), _sz(B), ctypes.c_int(k1))
    return out


def tgsw_external_mul_k(accum, bk_row):
    """Returns bk_row (x) accum for accum (B, k+1, N) and bk_row (k+1, 2, k+1, N), any mask size k <= 7."""
    out = _c(accum, numpy.int32).copy()
    bk_row = _c(bk_row, numpy.uint64)
    k1 = bk_row.shape[0]
    assert k1 <= 8 and out.shape[-2] == k1
    lib().orc_tgsw_external_mul_k(_p(out), _p(bk_row), _sz(out.size // (k1 * N)), ctypes.c_int(k1))
    return out


def bootstrap_k(in_a, in_b, bk, ks=None, mu=MU):
    """bootstrap() on the multi-kernel path for any mask size k (bootstrap.py:96-229), composed from the restated
    steps: bk (n, k+1, 2, k+1, N) in the reference's layout, ks for input size k * N.  Returns the key-switched sample
    (or the extracted one when ks is None) and the final accumulator."""
    in_a = _c(in_a, numpy.int32)
    in_b = _c(in_b, numpy.int32)
    bk = _c(bk, numpy.uint64)
    B, n, k1 = in_b.size, in_a.shape[-1], bk.shape[1]
    barb = t32_to_phase(in_b.reshape(B), 2 * N)
    bara = t32_to_phase(in_a.reshape(B, n), 2 * N)
    testvect = numpy.full((B, 1, N), mu, numpy.int32)
    acc = numpy.zeros((B, k1, N), numpy.int32)
    acc[:, k1 - 1, :] = shift_torus_polynomial(testvect, barb, invert_powers=True)[:, 0, :]
    for i in range(n):
        tmp = shift_torus_polynomial(acc, bara, i, minus_one=True)
        tmp = tgsw_external_mul_k(tmp, bk[i])
        acc = (acc.view(numpy.uint32) + tmp.view(numpy.uint32)).view(numpy.int32)
    ext_a = numpy.empty((B, k1 - 1, N), numpy.int32)
    ext_a[:, :, 0] = acc[:, :k1 - 1, 0]
    ext_a[:, :, 1:] = (0 - acc[:, :k1 - 1, :0:-1].view(numpy.uint32)).view(numpy.int32)
    ext_a = ext_a.reshape(B, (k1 - 1) * N)
    ext_b = numpy.ascontiguousarray(acc[:, k1 - 1, 0])
    if ks is None:
        return (ext_a, ext_b), acc
    ra, rb, _ = lwe_keyswitch(ks[0], ks[1], ks[2], ext_a, ext_b)
    return (ra, rb), acc


def blind_rotate(acc, bk, bara):
    out = _c(acc, numpy.int32).copy()
    bk = _c(bk, numpy.uint64)
    bara = _c(bara, numpy.int32)
    B = out.size // (2 * N)
    n = bara.size // B
    lib().orc_blind_rotate(_p(out), _p(bk), _p(bara), _sz(n), _sz(B))
    return out


def blind_rotate_mb(acc, bk, bara):
    """The multi-bit blind rotation (orc_blind_rotate_mb): acc (B, 2, N), bara (B, n) in [0, 2N) with n even, bk the
    multi-bit key's 3n/2 (or more) rows in the reference's transformed form (B, 2, 2, 2, N) uint64."""
    out = _c(acc, numpy.int32).copy()
    bk = _c(bk, numpy.uint64)
    bara = _c(bara, numpy.int32)
    B = out.size // (2 * N)
    n = bara.size // B
    assert n % 2 == 0 and bk.size >= 3 * (n // 2) * 8 * N, (n, bk.shape)
    assert ((bara >= 0) & (bara < 2 * N)).all()
    lib().orc_blind_rotate_mb(_p(out), _p(bk), _p(bara), _sz(n), _sz(B))
    return out


def lwe_keyswitch(ks_a, ks_b, ks_cv, src_a, src_b):
    ks_a = _c(ks_a, numpy.int32)
    ks_b = _c(ks_b, numpy.int32)
    ks_cv = _c(ks_cv, numpy.float32)
    src_a = _c(src_a, numpy.int32)
    src_b = _c(src_b, numpy.int32)
    input_size, t, base, output_size = ks_a.shape
    B = src_b.size
    res_a = numpy.empty(src_b.shape + (output_size,), numpy.int32)
    res_b = numpy.empty(src_b.shape, numpy.int32)
    res_cv = numpy.empty(src_b.shape, numpy.float32)
    lib().orc_lwe_keyswitch(
        _p(res_a), _p(res_b), _p(res_cv), _p(ks_a), _p(ks_b), _p(ks_cv), _p(src_a), _p(src_b),
        _sz(B), _sz(input_size), _sz(output_size), ctypes.c_int(t),
        ctypes.c_int(int(numpy.log2(base))))
    return res_a, res_b, res_cv


def bootstrap(in_a, in_b, bk, ks=None, mu=MU):
    """bootstrap(), nufhe/bootstrap.py:206-229.  ks = (ks_a, ks_b, ks_cv) or None (no_keyswitch)."""
    in_a = _c(in_a, numpy.int32)
    in_b = _c(in_b, numpy.int32)
    bk = _c(bk, numpy.uint64)
    B = in_b.size
    n = in_a.shape[-1]
    if ks is None:
        out_a = numpy.empty(in_b.shape + (N,), numpy.int32)
        ks_a = ks_b = ks_cv = None
        t = lb = 0
    else:
        ks_a = _c(ks[0], numpy.int32)
        ks_b = _c(ks[1], numpy.int32)
        ks_cv = _c(ks[2], numpy.float32)
        t, lb = ks_a.shape[1], int(numpy.log2(ks_a.shape[2]))
        out_a = numpy.empty(in_b.shape + (n,), numpy.int32)
    out_b = numpy.empty(in_b.shape, numpy.int32)
    lib().orc_bootstrap(
        _p(out_a), _p(out_b), _p(in_a), _p(in_b), _p(bk),
        _p(ks_a) if ks is not None else None, _p(ks_b) if ks is not None else None,
        _p(ks_cv) if ks is not None else None,
        ctypes.c_int32(int(mu)), _sz(B), _sz(n), ctypes.c_int(t), ctypes.c_int(lb))
    return out_a, out_b


# Linear prologues of the bootstrapped binary gates: t = (0, c/8) + sa*a + sb*b,
# nufhe/gates.py:81-597 (table in SURVEY.md section 8 a1).
GATE_TABLE = {
    'nand': (1, 8, -1, -1),
    'or': (1, 8, 1, 1),
    'and': (-1, 8, 1, 1),
    'xor': (1, 4, 2, 2),
    'xnor': (-1, 4, -2, -2),
    'nor': (-1, 8, -1, -1),
    'andny': (-1, 8, -1, 1),
    'andyn': (-1, 8, 1, -1),
    'orny': (1, 8, -1, 1),
    'oryn': (1, 8, 1, -1),
}


def phase_to_t32(phase, mspace_size):
    """numeric_functions.py:30-31"""
    v = (phase % mspace_size) * (2**32 // mspace_size)
    return numpy.int32(v - 2**32 if v >= 2**31 else v)


def lwe_affine2(a, b, c, sa, sb):
    a_a, a_b = a
    b_a, b_b = b
    with numpy.errstate(over='ignore'):
        t_a = (numpy.int32(sa) * a_a.astype(numpy.int32) + numpy.int32(sb) * b_a.astype(numpy.int32))
        t_b = (numpy.int32(c) + numpy.int32(sa) * a_b.astype(numpy.int32)
               + numpy.int32(sb) * b_b.astype(numpy.int32))
    return t_a.astype(numpy.int32), t_b.astype(numpy.int32)


def gate_binary(name, a, b, bk, ks):
    """gate_<name>(a, b) for the ten bootstrapped binary gates; a, b = (a_arr, b_arr) tuples."""
    num, den, sa, sb = GATE_TABLE[name]
    t_a, t_b = lwe_affine2(a, b, phase_to_t32(num, den), sa, sb)
    return bootstrap(t_a, t_b, bk, ks, MU)


def gate_mux(a, b, c, bk, ks):
    """gate_mux, nufhe/gates.py:600-664"""
    and_const = phase_to_t32(-1, 8)
    t_a, t_b = lwe_affine2(a, b, and_const, 1, 1)
    u1 = bootstrap(t_a, t_b, bk, None, MU)
    t_a, t_b = lwe_affine2(a, c, and_const, -1, 1)
    u2 = bootstrap(t_a, t_b, bk, None, MU)
    s_a, s_b = lwe_affine2(u1, u2, phase_to_t32(1, 8), 1, 1)
    r_a, r_b, _ = lwe_keyswitch(ks[0], ks[1], ks[2], s_a, s_b)
    return r_a, r_b


# ---------------------------------------------------------------- keys (reference RNG order)

def double_to_t32(d):
    """numeric_functions.py:39-40"""
    return ((d - numpy.trunc(d)) * 2**32).astype(numpy.int32)


def poly_mul_i32(a, b):
    a = _c(a, numpy.int32)
    b = _c(b, numpy.int32)
    out = numpy.empty_like(b)
    lib().orc_poly_mul_i32(_p(out), _p(a), _p(b), _sz(b.size // N))
    return out


def bk_transform(raw):
    """Bootstrap-key polynomials (..., N) int32 -> the reference's form: NTT, Montgomery (tgsw_transform_samples,
    tlwe_gpu.py:199-236); linear over the field, so keys with coefficients outside int32 are sums of two transforms."""
    raw = _c(raw, numpy.int32)
    out = numpy.empty(raw.shape, numpy.uint64)
    lib().orc_bk_transform(_p(out), _p(raw), _sz(_batch(raw)))
    return out


class OracleKeys:
    """Secret + cloud key material as host arrays, drawn in the reference's order from a seed."""

    def __init__(self, seed, n=LWE_N, make_bk=True, mask_size=1):
        rng = numpy.random.RandomState(seed)
        self.rng = rng
        self.n = n
        k = self.mask_size = mask_size
        # (1) LWE key, lwe.py:77-79
        self.lwe_key = rng.randint(0, 2, size=(n,), dtype=numpy.int32)
        # (2) TLWE key, tlwe.py:83-92
        self.tlwe_key = rng.randint(0, 2, size=(k, N), dtype=numpy.int32)
        if not make_bk:
            return
        # (3) bootstrap key: tlwe_encrypt_zero (tlwe.py:184-197) on shape (n, k+1, 2)
        noises1 = rng.randint(-2**31, 2**31, size=(n, k + 1, 2, k, N), dtype=numpy.int32)
        noises2 = double_to_t32(rng.normal(size=(n, k + 1, 2, N), scale=BS_STDEV))
        with numpy.errstate(over='ignore'):
            body = noises2.copy()
            for i in range(k):                                                   # tlwe_cpu.py:76-86
                body = body + poly_mul_i32(self.tlwe_key[i], numpy.ascontiguousarray(noises1[:, :, :, i, :]))
        bk = numpy.empty((n, k + 1, 2, k + 1, N), numpy.int32)
        bk[:, :, :, :k, :] = noises1
        bk[:, :, :, k, :] = body
        # tgsw_add_message, tgsw_cpu.py:109-126: += s_i * 2^(32-10(j+1)) on the diagonal, coefficient 0
        base_powers = numpy.array([2**22, 2**12], numpy.int32)
        with numpy.errstate(over='ignore'):
            for mi in range(k + 1):
                bk[:, mi, :, mi, 0] += self.lwe_key[:, None] * base_powers[None, :]
        self.bk_raw = bk
        # tgsw_transform_samples: NTT + Montgomery form (tlwe_gpu.py:199-236)
        self.bk = bk_transform(bk)
        # (4) key-switch key, lwe.py:265-295 + lwe_cpu.py:26-59; input size k * N
        t, base = KS_T, 2**KS_LOG2_BASE
        size_in = k * N
        noises_b = rng.normal(size=(size_in, t, base - 1), scale=KS_STDEV)
        noises_b -= noises_b.mean()
        noises_b = double_to_t32(noises_b)
        noises_a = rng.randint(-2**31, 2**31, size=(size_in, t, base - 1, n), dtype=numpy.int32)
        in_key = self.tlwe_key.ravel()
        hs = numpy.arange(1, base).astype(numpy.int32)
        js = numpy.arange(t).astype(numpy.int32)
        with numpy.errstate(over='ignore'):
            messages = (in_key[:, None, None] * hs[None, None, :]
                        * (2**(32 - (js[None, :, None] + 1) * KS_LOG2_BASE)).astype(numpy.int32))
        dot = numpy.empty((size_in, t, base - 1), numpy.int32)
        lib().orc_lwe_dot(_p(dot), _p(noises_a), _p(self.lwe_key), _sz(size_in * t * (base - 1)), _sz(n))
        self.ks_a = numpy.zeros((size_in, t, base, n), numpy.int32)
        self.ks_b = numpy.zeros((size_in, t, base), numpy.int32)
        self.ks_cv = numpy.zeros((size_in, t, base), numpy.float32)
        self.ks_a[:, :, 1:, :] = noises_a
        with numpy.errstate(over='ignore'):
            self.ks_b[:, :, 1:] = (messages.astype(numpy.int32) + noises_b + dot)
        self.ks_cv[:, :, 1:] = KS_STDEV**2

    @property
    def ks(self):
        return self.ks_a, self.ks_b, self.ks_cv

    def encrypt(self, bits):
        """encrypt(), api_low_level.py:266-281 + lwe.py:325-333 + lwe_cpu.py:104-112"""
        bits = numpy.asarray(bits).astype(bool)
        mus = numpy.where(bits, MU, -MU).astype(numpy.int32)
        noises_b = double_to_t32(self.rng.normal(size=bits.shape, scale=KS_STDEV))
        a = self.rng.randint(-2**31, 2**31, size=bits.shape + (self.n,), dtype=numpy.int32)
        dot = numpy.empty(bits.shape, numpy.int32)
        lib().orc_lwe_dot(_p(dot), _p(a), _p(self.lwe_key), _sz(bits.size), _sz(self.n))
        with numpy.errstate(over='ignore'):
            b = (noises_b + mus + dot).astype(numpy.int32)
        return a, b

    def decrypt(self, ct, key=None):
        """decrypt(), api_low_level.py:284-295"""
        a, b = ct
        key = self.lwe_key if key is None else key
        a = _c(a, numpy.int32)
        b = _c(b, numpy.int32)
        ph = numpy.empty(b.shape, numpy.int32)
        lib().orc_lwe_phase(_p(ph), _p(a), _p(b), _p(_c(key, numpy.int32)), _sz(b.size), _sz(a.shape[-1]))
        return ph > 0

    def phase(self, ct, key=None):
        a, b = ct
        key = self.lwe_key if key is None else key
        a = _c(a, numpy.int32)
        b = _c(b, numpy.int32)
        ph = numpy.empty(b.shape, numpy.int32)
        lib().orc_lwe_phase(_p(ph), _p(a), _p(b), _p(_c(key, numpy.int32)), _sz(b.size), _sz(a.shape[-1]))
        return ph
