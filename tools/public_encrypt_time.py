"""Time public-key encryption on one GPU with CUDA events over `--reps` calls after a warm-up: nb_pk_encrypt alone and
the whole ctx.encrypt(pk, bits) at B = 1, 4096 and 65 536, and nb_pk_prepare once.  Prints the card (name, power
limit, max SM clock, read in the same run) and the kernel's integer-op rate, 2 B m 4 N_padded (the four byte-plane
GEMMs), as a share of the H100 SXM data-sheet 1 979 TOPS dense INT8.

    python tools/public_encrypt_time.py [--reps 20]
"""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

INT8_OPS_PER_S = 1979e12


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
        sys.exit('public_encrypt_time.py needs a CUDA device')
    import numpy
    import nufhe_b200
    from nufhe_b200.engine import Engine
    from nufhe_b200.public_key import NONCE_ENCRYPTION_RANDOMNESS
    eng = Engine(0)
    print('card:', card())
    ctx = nufhe_b200.Context(rng=nufhe_b200.DeterministicRNG(1), thread=eng)
    sk = ctx.make_secret_key()
    pk = ctx.make_public_key(sk)
    m, n = pk.size, sk.params.in_out_params.size
    npad = (n + 2 + 7) // 8 * 8
    masks, body = pk.masks(eng), pk.b
    t = timed(lambda: eng.pk_prepare(masks, body), 1)
    print('nb_pk_prepare (m = %d, n = %d, %.1f MB of planes): %.3f ms'
          % (m, n, eng.lib.nb_pk_planes_bytes(m, n) / 1e6, t * 1e3))
    planes = pk.planes(eng)
    rng = numpy.random.RandomState(0)
    for batch in (1, 4096, 65536):
        r_words = eng.seeded_uniform(numpy.arange(8), NONCE_ENCRYPTION_RANDOMNESS, (batch, m // 32))
        mus = eng.to_device(rng.randint(-2**31, 2**31, batch, dtype=numpy.int64).astype(numpy.int32))
        t = timed(lambda: eng.public_encrypt(r_words, planes, m, n, mus, pk.variance), args.reps)
        ops = 2.0 * batch * m * 4 * npad
        bits = rng.randint(0, 2, batch).astype(bool)
        t_all = timed(lambda: ctx.encrypt(pk, bits), args.reps)
        print('B = %5d: nb_pk_encrypt %.3f ms (%.1f G int ops, %.1f TOPS, %.1f %% of 1979 TOPS INT8); '
              'ctx.encrypt(pk, bits) %.3f ms (%.0f bits/s)'
              % (batch, t * 1e3, ops / 1e9, ops / t / 1e12, 100 * ops / t / INT8_OPS_PER_S, t_all * 1e3,
                 batch / t_all))


if __name__ == '__main__':
    main()
