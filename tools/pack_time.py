"""Time result packing on one GPU with CUDA events over `--reps` calls after a warm-up, at B = 4096 and 65 536 gate
outputs: each step of one packing pass (nb_pack_digits, the forward NTT of the digits, nb_ntt_mac, the inverse NTT,
nb_pack_finish), their sum over the passes of a call as the kernel time, and the whole vm.pack call.  Prints the card
(name, power limit, max SM clock, read in the same run) and the HBM bytes each step has to move at least.

    python tools/pack_time.py [--reps 20]
"""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


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
        sys.exit('pack_time.py needs a CUDA device')
    import numpy
    import nufhe_b200
    from nufhe_b200.engine import Engine
    from nufhe_b200.packing import groups_per_pass
    eng = Engine(0)
    print('card:', card())
    ctx = nufhe_b200.Context(rng=nufhe_b200.DeterministicRNG(1), thread=eng)
    sk = ctx.make_secret_key()
    vm = ctx.make_virtual_machine(ctx.make_cloud_key(sk))
    psk, pk = ctx.make_packing_keys(sk)
    n, N = sk.params.in_out_params.size, 1024
    key = pk.spectra(eng)
    R, U = key.shape[0], key.shape[1]
    print('packing key spectra: %d x %d polynomials, %.1f MB; %d groups per pass'
          % (R, U, key.numel() * 8 / 1e6, groups_per_pass(sk.params)))
    rng = numpy.random.RandomState(0)
    for batch in (4096, 65536):
        x, y = rng.randint(0, 2, (2, batch)).astype(bool)
        r = vm.gate_nand(ctx.encrypt(sk, x), ctx.encrypt(sk, y))
        G = -(-batch // N)
        step = min(G, groups_per_pass(sk.params))
        a, b = r.a[:step * N].contiguous(), r.b[:step * N].contiguous()
        digits = eng.pack_digits(a)
        spec = eng.ntt_forward_i32(digits)
        prod = eng.ntt_mac(spec, key)
        c = eng.ntt_inverse_i32(prod)
        steps = [('nb_pack_digits', lambda: eng.pack_digits(a), a.numel() * 4 + digits.numel() * 4),
                 ('ntt_forward_i32', lambda: eng.ntt_forward_i32(digits), digits.numel() * 12),
                 ('nb_ntt_mac', lambda: eng.ntt_mac(spec, key), spec.numel() * 8 + key.numel() * 8 + prod.numel() * 8),
                 ('ntt_inverse_i32', lambda: eng.ntt_inverse_i32(prod), prod.numel() * 12),
                 ('nb_pack_finish', lambda: eng.pack_finish(c, b), c.numel() * 6 + b.numel() * 4)]
        passes = -(-G // step)
        total = 0.0
        print('B = %d: %d groups, %d pass(es) of %d groups' % (batch, G, passes, step))
        for name, fn, nbytes in steps:
            t = timed(fn, args.reps)
            total += t * passes
            print('  %-16s %.4f ms per pass (%.1f MB, %.2f TB/s)' % (name, t * 1e3, nbytes / 1e6, nbytes / t / 1e12))
        packed = vm.pack(pk, r)
        assert (ctx.decrypt(psk, packed) == ~(x & y)).all()
        t_all = timed(lambda: vm.pack(pk, r), args.reps)
        print('  kernel time %.3f ms; vm.pack %.3f ms (%.0f bits/s); pickle %d bytes'
              % (total * 1e3, t_all * 1e3, batch / t_all, len(packed.dumps())))


if __name__ == '__main__':
    main()
