"""Time the seeded-mask expansion (nb_seeded_uniform_i32) and a full cloud-key decompress() on one GPU, with CUDA
events after a warm-up.  Prints the card (name, power limit, max SM clock, read in the same run), the time, the write
rate in GB/s and its share of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s) -- the kernel only writes.

    python tools/seeded_expand_time.py [--reps 20]
"""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_BYTES_PER_S = 3.35e12


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True).stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0)


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e-3


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    ap.add_argument('--reps', type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('seeded_expand_time.py needs a CUDA device')
    import numpy
    import nufhe_b200
    from nufhe_b200.engine import Engine
    eng = Engine(0)
    print('card:', card())
    seed = numpy.arange(8, dtype=numpy.uint32) * 0x9e3779b9
    for name, shape in (('KS-key mask (1024, 8, 4, 500)', (1024, 8, 4, 500)),
                        ('65536-ciphertext mask (65536, 500)', (65536, 500))):
        out = torch.empty(shape, dtype=torch.int32, device=eng.device)
        words = out.numel()

        def expand():
            eng._call('nb_seeded_uniform_i32', seed.ctypes.data_as(nufhe_b200._native.ctypes.c_void_p), 2, 0,
                      nufhe_b200.engine._ptr(out), words)
        t = timed(expand, args.reps)
        rate = 4 * words / t
        print('%s: %d words, %.1f MB, %.3f ms, %.0f GB/s written, %.1f %% of 3.35 TB/s'
              % (name, words, 4 * words / 1e6, t * 1e3, rate / 1e9, 100 * rate / HBM_BYTES_PER_S))
    ctx = nufhe_b200.Context(rng=nufhe_b200.DeterministicRNG(1), thread=eng)
    sk = ctx.make_secret_key()
    cck = ctx.make_cloud_key(sk, compressed=True)
    t = timed(lambda: cck.decompress(eng), max(3, args.reps // 4))
    print('CompressedCloudKey.decompress(): %.2f ms (%.1f MB -> %.1f MB serialized)'
          % (t * 1e3, len(cck.dumps()) / 1e6, len(cck.decompress(eng).dumps()) / 1e6))


if __name__ == '__main__':
    main()
