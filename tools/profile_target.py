"""Small fixed workload for ncu captures: one blind-rotate launch (B ciphertexts), one key switch, a batch
of stand-alone transforms.  Usage: python tools/profile_target.py [B] [n_transforms]"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch                                   # noqa: E402
from nufhe_b200.engine import Engine           # noqa: E402

B = int(sys.argv[1]) if len(sys.argv) > 1 else 592
NT = int(sys.argv[2]) if len(sys.argv) > 2 else 65536
eng = Engine(0)
g = torch.Generator(device='cpu').manual_seed(7)


def rnd32(shape):
    return torch.randint(-2**31, 2**31, shape, generator=g, dtype=torch.int64).to(torch.int32).cuda()


def integral_bk(shape):
    # a bootstrap key whose polynomials are centred 32-bit integers, in the reference's form (NTT, Montgomery), as
    # real keys are: nb_bk_prepare gives it spectra, so the launch below runs the FP64 step that bench.py times.  (A
    # key of random field elements has no spectra and would time the NTT step.)
    from oracle import oracle as O
    raw = torch.randint(-2**31, 2**31, shape, generator=g, dtype=torch.int64).to(torch.int32).numpy()
    return torch.from_numpy(O.bk_transform(raw).view('int64')).cuda()


bk_int = eng.bk_prepare(integral_bk((500, 2, 2, 2, 1024)))
ks = (rnd32((1024, 8, 4, 500)), rnd32((1024, 8, 4)), torch.zeros((1024, 8, 4), dtype=torch.float32).cuda())
x1 = (rnd32((B, 500)), rnd32((B,)))
x2 = (rnd32((B, 500)), rnd32((B,)))
polys = rnd32((NT, 1024))


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return out, e0.elapsed_time(e1)


for it in range(3):
    ext, t_br = timed(lambda: eng.bootstrap_extract(x1, x2, 2**29, -1, -1, 2**29, bk_int))
    res, t_ks = timed(lambda: eng.keyswitch(ks, ext))
    f, t_f = timed(lambda: eng.ntt_forward_i32(polys))
    r, t_i = timed(lambda: eng.ntt_inverse_i32(f))
    assert bool((r == polys).all())
print('checksum', int(ext[0].to(torch.int64).sum()), int(res[0].to(torch.int64).sum()))
print('TIMES B=%d: blind_rotate %.3f ms (%.1f ns/ct-step), keyswitch %.3f ms, ntt_fwd %.3f ms (%.1f GB/s), '
      'ntt_inv %.3f ms (%.1f GB/s)' % (B, t_br, t_br * 1e6 / (B * 500), t_ks, t_f, NT * 12288 / t_f / 1e6,
                                       t_i, NT * 12288 / t_i / 1e6))
print('profile target done', eng.build_info())
