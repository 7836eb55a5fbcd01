#!/usr/bin/env python
"""Time the multi-key gate (nb_mk_bootstrap_extract + nb_mk_keyswitch, DESIGN.md section 17) against a loop over the
tenants that issues what each tenant's VirtualMachine.gate_nand issues (nb_bootstrap_extract + nb_keyswitch with that
tenant's key), alternated in one process, with CUDA events.

    python tools/multikey_time.py [--keys 128] [--reps 5] [--mixes 2048x1,256x16,64x64,16x256,1x4096] [--json PATH]

Tenant t uses key t % K of K distinct keys: K engine bootstrap keys (nb_bk_prepare of one reference key, K times, so
each lies at its own address) and K copies of one key-switch key, the first registered for the tensor-core key switch
as VirtualMachine does.  Key material does not change the work, only which memory is read.  The card's name, power
limit and SM clock limit are read in the same run.  Prints one line per mix and one JSON object at the end.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FFT_ROW_BYTES = 16 * 512 * 16          # the FP64 part of an engine key row (8 polynomials x 2 halves of 512 complex)


def gpu_info():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return out
    except Exception as e:                      # noqa: BLE001 - informational only
        return 'nvidia-smi unavailable (%s)' % e


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        start.record()
        fn()
        end.record()
        end.synchronize()
        ts.append(start.elapsed_time(end))
    return ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--keys', type=int, default=128, help='distinct keys the tenants cycle through')
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--mixes', default='2048x1,256x16,64x64,16x256,1x4096')
    ap.add_argument('--json', default=None, help='also write the results to this file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('multikey_time.py measures on a CUDA device; there is none')
    from oracle import oracle as O
    from nufhe_b200.engine import Engine

    eng = Engine(0)
    ref = O.OracleKeys(20261017)
    bk_ref = eng.to_device(ref.bk)
    K = args.keys
    bks = [eng.bk_prepare(bk_ref) for _ in range(K)]
    ks0 = tuple(eng.to_device(x) for x in ref.ks)
    kss = [ks0] + [tuple(x.clone() for x in ks0) for _ in range(K - 1)]
    planes = eng.ks_prepare(ks0[0], ks0[1])
    assert planes is not None
    torch.cuda.synchronize()
    info = gpu_info()
    print('device:', torch.cuda.get_device_name(0), '|', info, '| keys:', K, flush=True)

    c, s, mu = O.phase_to_t32(1, 8), -1, O.MU
    rng = numpy.random.RandomState(1)
    results = []
    for mix in args.mixes.split(','):
        T, per = (int(v) for v in mix.split('x'))
        B = T * per
        x1 = (eng.to_device(rng.randint(-2**31, 2**31, size=(B, 500), dtype=numpy.int32)),
              eng.to_device(rng.randint(-2**31, 2**31, size=(B,), dtype=numpy.int32)))
        x2 = (eng.to_device(rng.randint(-2**31, 2**31, size=(B, 500), dtype=numpy.int32)),
              eng.to_device(rng.randint(-2**31, 2**31, size=(B,), dtype=numpy.int32)))
        counts = [per] * T
        tb = [bks[t % K] for t in range(T)]
        tk = [kss[t % K] for t in range(T)]
        out = {}

        def multi():
            ext = eng.mk_bootstrap_extract(x1, x2, c, s, s, mu, tb, counts)
            out['mk'] = eng.mk_keyswitch(tk, counts, ext, want_cv=True)

        def multi_bootstrap():
            eng.mk_bootstrap_extract(x1, x2, c, s, s, mu, tb, counts)

        def loop():
            res = []
            for t in range(T):
                lo, hi = t * per, (t + 1) * per
                ext = eng.bootstrap_extract((x1[0][lo:hi], x1[1][lo:hi]), (x2[0][lo:hi], x2[1][lo:hi]), c, s, s, mu, tb[t])
                res.append(eng.keyswitch(tk[t], ext, want_cv=True))
            out['loop'] = res

        for fn in (multi, loop, multi_bootstrap):          # warm-up: modules, scratch buffers
            fn()
        torch.cuda.synchronize()
        got, want = out['mk'], out['loop']
        same = all(torch.equal(got[i], torch.cat([r[i] for r in want])) for i in range(3))
        t_mk, t_loop, t_br = [], [], []
        for _ in range(args.reps):                          # alternated
            t_mk += timed(multi, 1)
            t_loop += timed(loop, 1)
            t_br += timed(multi_bootstrap, 1)
        med = lambda v: float(numpy.median(v))
        key_bytes = B * 500 * FFT_ROW_BYTES                 # key rows a ciphertext's chain streams (no reuse between chains)
        row = {'mix': mix, 'tenants': T, 'per_tenant': per, 'bit_identical': bool(same),
               'multi_ms': med(t_mk), 'multi_ms_range': [min(t_mk), max(t_mk)],
               'loop_ms': med(t_loop), 'loop_ms_range': [min(t_loop), max(t_loop)],
               'multi_bootstrap_ms': med(t_br), 'speedup': med(t_loop) / med(t_mk),
               'key_stream_gb': key_bytes / 1e9, 'key_stream_tb_s': key_bytes / (med(t_br) * 1e-3) / 1e12}
        results.append(row)
        print('%-8s multi %8.2f ms [%6.2f, %6.2f]  loop %9.2f ms [%8.2f, %8.2f]  x%6.2f  bootstrap %8.2f ms  '
              'key stream %6.1f GB = %5.2f TB/s  identical=%s' % (
                  mix, row['multi_ms'], min(t_mk), max(t_mk), row['loop_ms'], min(t_loop), max(t_loop), row['speedup'],
                  row['multi_bootstrap_ms'], row['key_stream_gb'], row['key_stream_tb_s'], same), flush=True)
        del x1, x2, out
    summary = {'device': torch.cuda.get_device_name(0), 'nvidia_smi': info, 'keys': K, 'reps': args.reps,
               'time': time.strftime('%Y-%m-%d %H:%M:%S'), 'results': results}
    print(json.dumps(summary))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(summary, f, indent=1)


if __name__ == '__main__':
    main()
