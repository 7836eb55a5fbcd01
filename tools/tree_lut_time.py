#!/usr/bin/env python
"""Time tree-based LUTs (nufhe_b200/tree_lut.py) on one GPU with CUDA events: each step of a level >= 2 at B = 4096
tree test vectors (nb_tree_keyswitch, nb_tree_assemble, nb_bootstrap_glwe_lut_extract, the key switch), the one-output
LUT bootstrap (nb_bootstrap_lut_extract) at the same batch for comparison, and whole vm.lut_tree calls on 4096
ciphertexts at P = 2, D = 2 and D = 4.  Prints the card and one JSON line.

    python tools/tree_lut_time.py [--batch 4096] [--reps 5] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import nufhe_b200  # noqa: E402
from nufhe_b200.tgsw import engine_format  # noqa: E402


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True).stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0)


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    return float(numpy.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=4096)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    print('card:', card())
    ctx = nufhe_b200.Context(rng=nufhe_b200.DeterministicRNG(7))
    sk = ctx.make_secret_key()
    ck, tk = ctx.make_cloud_key(sk, tree_key=True)
    vm = ctx.make_virtual_machine(ck)
    thr = ctx.thread
    bk, ks = ck.bootstrap_key, ck.keyswitch_key
    bk_int = engine_format(thr, bk.tgsw)
    B, M = args.batch, 4
    rng = numpy.random.RandomState(1)
    res = {'card': card(), 'batch': B}

    # one level >= 2 at P = 2: B test vectors from 4 B LWE samples, rotated by B digits
    lv = ctx.encrypt_int(sk, rng.randint(0, 4, (B * M,)), 2)
    x = ctx.encrypt_int(sk, rng.randint(0, 4, (B,)), 2)
    planes = tk.planes(thr)
    v = thr.tree_keyswitch(lv.a, planes, 1)
    tv = thr.tree_assemble(v.reshape(B, M, 2, -1), lv.b.reshape(B, M), 2)
    ea, eb = thr.bootstrap_glwe_lut_extract((x.a, x.b), tv, bk_int)
    res['tree_keyswitch_ms'] = timed(lambda: thr.tree_keyswitch(lv.a, planes, 1), args.reps)
    res['tree_assemble_ms'] = timed(lambda: thr.tree_assemble(v.reshape(B, M, 2, -1), lv.b.reshape(B, M), 2), args.reps)
    res['glwe_lut_bootstrap_ms'] = timed(lambda: thr.bootstrap_glwe_lut_extract((x.a, x.b), tv, bk_int), args.reps)
    res['keyswitch_ms'] = timed(lambda: thr.keyswitch(ks.device_arrays(), (ea, eb)), args.reps)
    tv1 = thr.to_device(nufhe_b200.make_test_vector(rng.randint(0, 4, (B, 4)), 2))
    res['lut_bootstrap_ms'] = timed(lambda: thr.bootstrap_lut_extract((x.a, x.b), None, 0, 1, 0, tv1, 0, bk_int),
                                    args.reps)
    for D in (2, 4):
        digits = [ctx.encrypt_int(sk, rng.randint(0, 4, (B,)), 2) for _ in range(D)]
        table = vm.make_tree_lut(rng.randint(0, 4, (4,) * D), 2, D)
        ms = timed(lambda: vm.lut_tree(tk, table, digits), max(1, args.reps // 2))
        res['lut_tree_D%d_ms' % D] = ms
        res['lut_tree_D%d_per_s' % D] = B / ms * 1e3
    print(json.dumps(res))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
