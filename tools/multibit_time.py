#!/usr/bin/env python
"""Standard against multi-bit bootstrap keys (DESIGN.md section 14), in one process on one card: gate_nand, gate_mux
and a one-output LUT at batches 1 .. 65536, the fused bootstrap kernel alone (Engine.bootstrap_extract /
bootstrap_lut_extract on device-resident operands) and the whole VM call (bootstrap + key switch).  CUDA events,
median of repeated calls after a warm-up; the two keys alternate call by call.  The card's name, power limit and SM
clock are read before and after the runs.

    python tools/multibit_time.py [--batches 1,16,...] [--reps 5] [--out results.json]
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
from nufhe_b200.gates import MU  # noqa: E402


def card():
    q = 'name,power.limit,clocks.sm,clocks.max.sm,clocks_throttle_reasons.active'
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=' + q, '--format=csv,noheader'],
                              capture_output=True, text=True).stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0)


def timed(fns, warmup, reps):
    """median milliseconds of each function, the functions alternated call by call"""
    for _ in range(warmup):
        for f in fns:
            f()
    times = [[] for _ in fns]
    for _ in range(reps):
        for i, f in enumerate(fns):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            f()
            e.record()
            e.synchronize()
            times[i].append(s.elapsed_time(e))
    return [float(numpy.median(t)) for t in times]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batches', default='1,16,64,256,1024,4096,16384,65536')
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    ctx = nufhe_b200.Context(rng=nufhe_b200.DeterministicRNG(2026))
    sk = ctx.make_secret_key()
    keys = {'standard': ctx.make_cloud_key(sk), 'multi_bit': ctx.make_cloud_key(sk, multi_bit=2)}
    vms = {k: ctx.make_virtual_machine(ck) for k, ck in keys.items()}
    bks = {k: engine_format(ctx.thread, ck.bootstrap_key.tgsw) for k, ck in keys.items()}
    thr = ctx.thread
    res = {'card_before': card(), 'rows': []}
    rng = numpy.random.RandomState(1)
    for B in [int(b) for b in args.batches.split(',')]:
        a, b, c = (ctx.encrypt(sk, rng.randint(0, 2, B).astype(bool)) for _ in range(3))
        xi = ctx.encrypt_int(sk, rng.randint(0, 4, B), 2)
        luts = {k: vm.make_lut([3, 2, 1, 0], 2) for k, vm in vms.items()}
        reps = args.reps if B <= 16384 else max(3, args.reps // 2)
        pa, pb = (a.a.contiguous(), a.b.contiguous()), (b.a.contiguous(), b.b.contiguous())
        pi = (xi.a.contiguous(), xi.b.contiguous())
        ops = {
            'gate_nand': ({k: (lambda vm=vm: vm.gate_nand(a, b)) for k, vm in vms.items()},
                          {k: (lambda bk=bk: thr.bootstrap_extract(pa, pb, 1 << 29, -1, -1, MU, bk)) for k, bk in bks.items()}),
            'gate_mux': ({k: (lambda vm=vm: vm.gate_mux(a, b, c)) for k, vm in vms.items()}, None),
            'lut1': ({k: (lambda vm=vm, k=k: vm.lut(luts[k], xi)) for k, vm in vms.items()},
                     {k: (lambda bk=bk, k=k: thr.bootstrap_lut_extract(pi, None, 0, 1, 0, luts[k].tv, 0, bk))
                      for k, bk in bks.items()}),
        }
        for op, (calls, kernels) in ops.items():
            row = {'op': op, 'batch': B}
            t = timed([calls['standard'], calls['multi_bit']], args.warmup, reps)
            row['call_ms'] = {'standard': t[0], 'multi_bit': t[1], 'speedup': t[0] / t[1]}
            if kernels:
                t = timed([kernels['standard'], kernels['multi_bit']], args.warmup, reps)
                row['kernel_ms'] = {'standard': t[0], 'multi_bit': t[1], 'speedup': t[0] / t[1]}
            res['rows'].append(row)
            print(json.dumps(row), flush=True)
    res['card_after'] = card()
    print(json.dumps({'card_before': res['card_before'], 'card_after': res['card_after']}))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
