"""A reference for multi-bit bootstrap keys (nufhe_b200/bootstrap.py: MultiBitBootstrapKey): key generation from an
OracleKeys' secrets and the multi-bit blind rotation, plus the entry points of the fused bootstrap composed with the
oracle's head and tail steps (as tests/fused_ref.py does for the standard key).  TEST INFRASTRUCTURE ONLY; it shares no
code with the CUDA source.

The rotation works on the keys' integer coefficients, not on their transformed form:

    ACC += sum_{p = 1..3} (X^{k_p} - 1) . (Dec(ACC) [x] BK_{g,p}),   k_1 = abar_2g, k_2 = abar_2g+1, k_3 = k_1 + k_2

Every product is an exact integer polynomial reduced mod 2^32.  It is computed with float64 FFTs in torch on 16-bit
halves of the key (coefficients below 6 x 2^36, so the rounding error of a length-1024 FFT is orders of magnitude
below 1/2), and every coefficient is checked to lie within 1/4 of an integer before it is rounded: a sanity check
that catches a reference drifting towards its precision limit, not a proof of exactness (an error above 3/4 would
pass it).  It is fast enough for large batches on the GPU (torch), but it is not exact.  The exact-integer oracle is the
C oracle's multi-bit rotation (`blind_rotate_oracle`, O.blind_rotate_mb, on the key's transformed rows): every
composition below takes the rotation as its `rotate` argument, so the same composition runs on either.  The two agree
bit for bit on noisy keys, random and edge rotations (tests/test_host_multibit.py); the same float machinery run as the
standard rotation (`blind_rotate_std`) gives the C oracle's bootstrap bit for bit, and with noiseless keys every
rotation gives the exact rotation."""
import numpy
import torch

from oracle import oracle as O

N = 1024


def indicators(lwe_key):
    """(3n/2,) int32: row 3 g + p - 1 holds [s_2g = b0 and s_2g+1 = b1], p = b0 + 2 b1"""
    s = numpy.asarray(lwe_key, numpy.int64).reshape(-1, 2)
    s0, s1 = s[:, 0], s[:, 1]
    return numpy.stack([s0 * (1 - s1), (1 - s0) * s1, s0 * s1], axis=1).reshape(-1).astype(numpy.int32)


def tgsw_rows(tlwe_key, messages, rng, noiseless=False):
    """TGSW encryptions (k = 1, l = 2, Bg = 2^10) of `messages` under tlwe_key (1, N): raw rows (R, 2, 2, 2, N) int32.
    noiseless: zero masks and zero noise, the trivial samples of the messages."""
    R = len(messages)
    if noiseless:
        bk = numpy.zeros((R, 2, 2, 2, N), numpy.int32)
    else:
        noises1 = rng.randint(-2**31, 2**31, size=(R, 2, 2, N), dtype=numpy.int32)
        noises2 = O.double_to_t32(rng.normal(size=(R, 2, 2, N), scale=O.BS_STDEV))
        with numpy.errstate(over='ignore'):
            body = noises2 + O.poly_mul_i32(tlwe_key[0], noises1)
        bk = numpy.stack([noises1, body], axis=3).astype(numpy.int32)
    base_powers = numpy.array([2**22, 2**12], numpy.int64)
    for mi in range(2):
        v = bk[:, mi, :, mi, 0].astype(numpy.int64) + numpy.asarray(messages, numpy.int64)[:, None] * base_powers
        bk[:, mi, :, mi, 0] = (v & 0xffffffff).astype(numpy.uint32).view(numpy.int32)
    return bk


def multibit_key(keys, seed, noiseless=False):
    """(raw rows (3n/2, 2, 2, 2, N) int32, the same in the reference's transformed form) for an OracleKeys' secrets"""
    raw = tgsw_rows(keys.tlwe_key, indicators(keys.lwe_key), numpy.random.RandomState(seed), noiseless)
    return raw, O.bk_transform(raw)


def standard_key(keys, seed, noiseless=False):
    """the standard key of the same secrets, raw and transformed"""
    raw = tgsw_rows(keys.tlwe_key, keys.lwe_key, numpy.random.RandomState(seed), noiseless)
    return raw, O.bk_transform(raw)


class _Fft:
    def __init__(self, device):
        self.device = device
        j = torch.arange(N, dtype=torch.float64, device=device)
        self.twist = torch.polar(torch.ones_like(j), torch.pi * j / N)                # w^j, w = e^{i pi / N}
        e = torch.arange(2 * N, dtype=torch.float64, device=device)
        self.roots = torch.polar(torch.ones_like(e), torch.pi * e / N)                # e^{2 pi i e / 2N}
        self.m = torch.arange(N, dtype=torch.int64, device=device)

    def fwd(self, x):
        """x (..., N) real -> its values at w^(1 - 2 m), m < N"""
        return torch.fft.fft(x.to(torch.float64) * self.twist, dim=-1)

    def inv(self, X):
        return (torch.fft.ifft(X, dim=-1) / self.twist).real

    def rotation(self, k):
        """the spectrum of X^k for k (B,): e^{i pi k (1 - 2 m) / N}"""
        return self.roots[(k[:, None] * (1 - 2 * self.m)[None, :]) % (2 * N)]

    def key(self, rows):
        """raw rows (P, 2 mi, 2 j, 2 mo, N) -> spectra (P, 4 d, 2 mo, 2 h, N) of the 16-bit halves"""
        k = torch.as_tensor(numpy.asarray(rows, numpy.int64), device=self.device)
        lo = ((k + 32768) & 65535) - 32768
        hi = (k - lo) >> 16
        return self.fwd(torch.stack([lo, hi], dim=-2)).reshape(k.shape[0], 4, 2, 2, N)


def _decompose(acc):
    """signed digits (B, 4 d = mi * 2 + j, N) of acc (B, 2, N) int64 (tgsw_gpu.mako; offset 2^31 + 2^21)"""
    t = (acc + (2**31 + 2**21)) & 0xffffffff
    return torch.stack([((t >> 22) & 1023) - 512, ((t >> 12) & 1023) - 512], dim=2).reshape(acc.shape[0], 4, N)


def _accumulate(F, acc, spec):
    """acc += the exact integer polynomials of spec (B, 2 mo, 2 h, N), halves recombined mod 2^32"""
    y = F.inv(spec)
    r = torch.round(y)
    err = (y - r).abs().max().item() if y.numel() else 0.0
    assert err < 0.25, 'the float64 reference is not exact here (%g)' % err
    r = r.to(torch.int64)
    return (acc + r[:, :, 0] + (r[:, :, 1] << 16)) & 0xffffffff


def _to_acc(acc, device):
    return torch.as_tensor(numpy.asarray(acc, numpy.int64) & 0xffffffff, device=device)


def _from_acc(acc):
    return (acc.cpu().numpy() & 0xffffffff).astype(numpy.uint32).view(numpy.int32)


def blind_rotate_mb(acc, bara, bk_raw, device='cpu'):
    """accum (B, 2, N) int32, bara (B, n) in [0, 2N), bk_raw (3n/2, 2, 2, 2, N): the multi-bit blind rotation"""
    F = _Fft(device)
    acc = _to_acc(acc, device)
    bara = torch.as_tensor(numpy.asarray(bara, numpy.int64), device=device)
    for g in range(bara.shape[1] // 2):
        D = F.fwd(_decompose(acc))                                                    # (B, 4, N)
        K = F.key(bk_raw[3 * g:3 * g + 3])
        a0, a1 = bara[:, 2 * g], bara[:, 2 * g + 1]
        out = 0
        for p, k in enumerate((a0, a1, (a0 + a1) % (2 * N))):
            S = torch.einsum('bdn,dohn->bohn', D, K[p])
            out = out + (F.rotation(k) - 1)[:, None, None, :] * S
        acc = _accumulate(F, acc, out)
    return _from_acc(acc)


def blind_rotate_oracle(acc, bara, bk_ref, device=None):
    """the exact-integer multi-bit rotation of the C oracle (O.blind_rotate_mb); bk_ref is the key in the reference's
    transformed form (the second value of multibit_key), not its raw rows"""
    return O.blind_rotate_mb(acc, bk_ref, bara)


def blind_rotate_std(acc, bara, bk_raw, device='cpu'):
    """the standard rotation through the same machinery: ACC += Dec((X^a_i - 1) ACC) [x] BK_i"""
    F = _Fft(device)
    acc = _to_acc(acc, device)
    bara = torch.as_tensor(numpy.asarray(bara, numpy.int64), device=device)
    idx = torch.arange(N, device=device)
    for i in range(bara.shape[1]):
        a = bara[:, i][:, None, None]
        # (X^a ACC)[x] = +-ACC[(x - a) mod N], minus where (x - a) mod 2N >= N
        src = (idx - a) % (2 * N)
        rot = torch.gather(acc, 2, (src % N).expand(acc.shape))
        rot = torch.where(src >= N, -rot, rot)
        D = F.fwd(_decompose((rot - acc) & 0xffffffff))
        S = torch.einsum('bdn,dohn->bohn', D, F.key(bk_raw[i:i + 1])[0])
        acc = _accumulate(F, acc, S)
    return _from_acc(acc)


def bootstrap_extract(x1, x2, c, s1, s2, mu, bk_raw, device='cpu', rotate=blind_rotate_mb):
    """the gate bootstrap without key switch (nb_bootstrap_extract) with a multi-bit key"""
    from fused_ref import prologue
    a, b = prologue(x1, x2, c, s1, s2)
    B = b.size
    tv = numpy.full((B, N), mu, numpy.int32)
    barb, bara = O.t32_to_phase(b, 2 * N), O.t32_to_phase(a, 2 * N)
    acc = O.tlwe_noiseless_trivial(O.shift_torus_polynomial(tv[:, None, :], barb, invert_powers=True)[:, 0])
    acc = rotate(acc, bara, bk_raw, device)
    return O.tlwe_extract_lwe_samples(acc)


def bootstrap_extract2(job_a, job_b, mu, bk_raw, device='cpu', rotate=blind_rotate_mb):
    ra = bootstrap_extract(*job_a, mu, bk_raw, device, rotate)
    rb = bootstrap_extract(*job_b, mu, bk_raw, device, rotate)
    return numpy.concatenate([ra[0], rb[0]]), numpy.concatenate([ra[1], rb[1]])


def bootstrap_lut_extract(x1, x2, c, s1, s2, tv, L, bk_raw, device='cpu', rotate=blind_rotate_mb):
    """the programmable bootstrap (nb_bootstrap_lut_extract) with a multi-bit key"""
    from fused_ref import prologue, _extract_outputs
    a, b = prologue(x1, x2, c, s1, s2)
    B = b.size
    barb = (O.t32_to_phase(b, (2 * N) >> L).astype(numpy.int64) << L).astype(numpy.int32)
    bara = (O.t32_to_phase(a, (2 * N) >> L).astype(numpy.int64) << L).astype(numpy.int32)
    tvs = numpy.ascontiguousarray(numpy.broadcast_to(numpy.asarray(tv).reshape(-1, N), (B, N)))
    acc = O.tlwe_noiseless_trivial(O.shift_torus_polynomial(tvs[:, None, :], barb, invert_powers=True)[:, 0])
    acc = rotate(acc, bara, bk_raw, device)
    return _extract_outputs(acc, L)


def bootstrap_glwe_lut_extract(x, tv, bk_raw, device='cpu', rotate=blind_rotate_mb):
    """nb_bootstrap_glwe_lut_extract with a multi-bit key"""
    from fused_ref import i32
    a, b = i32(x[0]), i32(x[1])
    barb, bara = O.t32_to_phase(b, 2 * N), O.t32_to_phase(a, 2 * N)
    acc = O.shift_torus_polynomial(numpy.asarray(tv, numpy.int32), barb, invert_powers=True)
    acc = rotate(acc, bara, bk_raw, device)
    return O.tlwe_extract_lwe_samples(acc)


def exact_rotation(tv, e):
    """X^e tv for tv (B, N) and e (B,): the body of a rotation by sum_i abar_i s_i with noiseless keys"""
    e = numpy.asarray(e, numpy.int64) % (2 * N)
    idx = numpy.arange(N)
    src = (idx[None, :] - e[:, None]) % (2 * N)
    v = numpy.take_along_axis(numpy.asarray(tv, numpy.int64), src % N, axis=1)
    v = numpy.where(src >= N, -v, v)
    return (v & 0xffffffff).astype(numpy.uint32).view(numpy.int32)
