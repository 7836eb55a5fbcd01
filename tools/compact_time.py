"""Time compact public-key encryption (DESIGN.md section 16) on one GPU at B = 1, 4096 and 65 536 messages:
`ctx.encrypt(cpk)` as a whole call and in its steps, `vm.expand` as a whole call and as its two steps (extraction, key
switch; each over the passes vm.expand makes), and `ctx.encrypt(pk)` with the section 11 public key for comparison.
CUDA events, median of --reps calls after --warmup.  Prints one JSON object with the card's name, power limit and SM
clocks, read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import numpy
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import nufhe_b200 as nufhe                      # noqa: E402
from nufhe_b200 import compact as C             # noqa: E402
from nufhe_b200.api_low_level import bool_to_t32                 # noqa: E402
from nufhe_b200.random_numbers import rand_gaussian_torus32      # noqa: E402

N = 1024


def median_ms(fn, warmup, reps):
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        times.append(s.elapsed_time(e))
    return float(numpy.median(times))


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm',
                              '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except Exception as e:            # (the figures are reported without a card line rather than not at all)
        return 'unknown (%s)' % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batches', type=int, nargs='*', default=[1, 4096, 65536])
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--out', help='also write the JSON object to this file')
    args = ap.parse_args()
    ctx = nufhe.Context(rng=nufhe.DeterministicRNG(1))
    sk = ctx.make_secret_key()
    ck, cpk = ctx.make_cloud_key(sk, compact_public_key=True)
    pub = ctx.make_public_key(sk)
    vm = ctx.make_virtual_machine(ck)
    thr = ctx.thread
    params = sk.params
    tl = params.tgsw_params.tlwe_params
    k = tl.mask_size
    ks = ck.keyswitch_key.device_arrays()
    res = {'card': card(), 'groups_per_pass': C.groups_per_pass(params), 'batches': {}}
    run = lambda fn: median_ms(fn, args.warmup, args.reps)         # noqa: E731
    for B in args.batches:
        bits = numpy.random.RandomState(B).randint(0, 2, B).astype(bool)
        G = -(-B // N)
        mus = thr.to_device(bool_to_t32(bits))
        r = {}
        r['encrypt_ms'] = run(lambda: ctx.encrypt(cpk, bits))
        # the steps of compact_encrypt
        r['encrypt_draws_ms'] = run(lambda: (rand_gaussian_torus32(thr, ctx.rng, 0, tl.min_noise, (G, k, N)),
                                             rand_gaussian_torus32(thr, ctx.rng, 0, tl.min_noise, (G, N))))
        seed = numpy.arange(8, dtype=numpy.uint32)
        r['encrypt_r_bits_ms'] = run(lambda: C.r_bits(thr, seed, G))
        rb = C.r_bits(thr, seed, G)
        r['encrypt_ntt_forward_ms'] = run(lambda: thr.ntt_forward_i32(rb))
        spec = thr.ntt_forward_i32(rb).reshape(G, 1, N)
        key = cpk.spectra(thr)
        r['encrypt_ntt_mac_ms'] = run(lambda: thr.ntt_mac(spec, key))
        mac = thr.ntt_mac(spec, key)
        r['encrypt_ntt_inverse_ms'] = run(lambda: thr.ntt_inverse_i32(mac))
        prod = thr.ntt_inverse_i32(mac)
        e1 = torch.zeros((G, k, N), dtype=torch.int32, device=thr.device)
        e2 = torch.zeros((G, N), dtype=torch.int32, device=thr.device)
        r['encrypt_finish_ms'] = run(lambda: thr.compact_finish(prod, e1, e2, mus))
        ct = ctx.encrypt(cpk, bits)
        r['ciphertext_bytes'] = len(ct.dumps())
        # vm.expand and its two steps, over the same passes
        r['expand_ms'] = run(lambda: vm.expand(ct))
        step = C.groups_per_pass(params) * N
        parts = [(c0, min(B, c0 + step)) for c0 in range(0, B, step)]
        data = ct.data
        r['expand_extract_ms'] = run(lambda: [thr.compact_extract(data[c0 // N:-(-c1 // N)], c1 - c0) for c0, c1 in parts])
        ext = [thr.compact_extract(data[c0 // N:-(-c1 // N)], c1 - c0) for c0, c1 in parts]
        r['expand_keyswitch_ms'] = run(lambda: [thr.keyswitch(ks, e, want_cv=True) for e in ext])
        # bytes the extraction writes (masks and bodies) and reads (the data)
        moved = B * (k * N + 1) * 4 + G * (k + 1) * N * 2
        r['extract_gb_per_s'] = moved / (r['expand_extract_ms'] * 1e-3) / 1e9
        del ext
        torch.cuda.empty_cache()
        # the section 11 public key
        r['public_key_encrypt_ms'] = run(lambda: ctx.encrypt(pub, bits))
        r['public_key_ciphertext_bytes'] = len(ctx.encrypt(pub, bits).dumps())
        assert (ctx.decrypt(sk, vm.expand(ct)) == bits).all()
        res['batches'][B] = r
        print(json.dumps({B: r}), flush=True)
    res['compact_public_key_bytes'] = len(cpk.dumps())
    res['public_key_bytes'] = len(pub.dumps())
    print(json.dumps(res))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
