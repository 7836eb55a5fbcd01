#!/usr/bin/env python
"""Time the multi-key machine on compressed cloud keys (resident_tenants, DESIGN.md section 19) with CUDA events.

    python tools/multikey_pool_time.py [--reps 5] [--tenants 2048] [--json PATH]

Keys are synthetic CompressedCloudKeys (random seeds and random bodies drawn on the device), ciphertexts random LWE
samples: the work and the bits computed do not depend on whether a secret key stands behind them.  Cells:
  expand R        nb_mk_bk_expand + nb_mk_ks_expand of R tenants into R slots (one launch each), per tenant, against
                  decompress() + engine_format of the same tenants one after the other; the slots' FP64 part and ks_a
                  must equal the decompressed keys' word for word;
  nand R          T distinct tenants x 1 NAND at R resident tenants: every call expands every tenant (the previous
                  call's residents first, in rounds of R); R = 128 and 256 must give the same bits, and sampled tenants
                  the bits of their decompressed VirtualMachine;
  resident 256x16 256 tenants x 16 NANDs at R = 256, second call (no expansion), against the machine on the same 256
                  keys decompressed and resident; the bits must agree.
Each cell: a warm-up, then the median and range of --reps runs.  The card's name, power limit and SM clock limit are
read in the same run.  Prints one line per cell and one JSON object at the end.
"""
import argparse
import gc
import json
import os
import subprocess
import sys

import numpy
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                      # noqa: BLE001 - informational only
        return 'nvidia-smi unavailable (%s)' % e


def timed(fn):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    out = fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end), out


def stats(fn, reps):
    timed(fn)                                   # warm-up
    times, out = [], None
    for _ in range(reps):
        ms, out = timed(fn)
        times.append(ms)
    return dict(median_ms=float(numpy.median(times)), min_ms=min(times), max_ms=max(times)), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--tenants', type=int, default=2048)
    ap.add_argument('--json', default=None, help='also write the JSON object to this file')
    args = ap.parse_args()

    import nufhe_b200
    from nufhe_b200.compressed import CompressedCloudKey
    from nufhe_b200.lwe import LweSampleArray
    from nufhe_b200.tgsw import engine_format

    ctx = nufhe_b200.Context(rng=nufhe_b200.DeterministicRNG(1))
    thr = ctx.thread
    params = nufhe_b200.NuFHEParameters()
    n = params.in_out_params.size
    dev = thr.device
    gen = torch.Generator(device=dev)
    gen.manual_seed(20261018)
    rng = numpy.random.RandomState(5)

    def i32(shape):
        return torch.randint(-2**31, 2**31, shape, dtype=torch.int32, device=dev, generator=gen)

    def key():
        seed = rng.randint(0, 2**32, size=8, dtype=numpy.int64).astype(numpy.uint32)
        return CompressedCloudKey(params, seed, i32((n, 2, 2, 1024)), 1e-9, i32((1024, 8, 4)), 2e-9)

    def samples(count, per):
        cv = lambda: torch.zeros((per,), dtype=torch.float32, device=dev)
        return [LweSampleArray(params.in_out_params, i32((per, n)), i32((per,)), cv()) for _ in range(count)]

    def same(x, y):
        return all(torch.equal(u, v) for u, v in ((x.a, y.a), (x.b, y.b), (x.current_variances, y.current_variances)))

    info = gpu_info()
    print('gpu:', info)
    cells = {}
    T = args.tenants
    keys = [key() for _ in range(T)]
    ntt = thr.lib.nb_bk_row_u64() - thr.lib.nb_bk_multibit_row_u64()

    # --- expansion alone
    for R in (64, 256):
        sub = keys[:R]
        slots = [thr.mk_bk_slot(n) for _ in range(R)]
        ks_as = [thr.empty((1024, 8, 4, n), torch.int32) for _ in range(R)]
        seeds = numpy.stack([k.seed for k in sub])

        def expand():
            thr.mk_bk_expand(seeds, [k.bk_body for k in sub], slots, params)
            thr.mk_ks_expand(seeds, ks_as)
        st, _ = stats(expand, args.reps)
        # the decompress path on the first 64 of the same tenants, one after the other (it holds one 250 MB key at a time)
        check = sub[:64]

        def decompress():
            for k in check:
                ck = k.decompress(thr)
                engine_format(thr, ck.bootstrap_key.tgsw)
        sd, _ = stats(decompress, args.reps)
        ok = True
        for i, k in enumerate(check[:8]):
            ck = k.decompress(thr)
            ok &= torch.equal(engine_format(thr, ck.bootstrap_key.tgsw)[:, ntt:], slots[i][:, ntt:])
            ok &= torch.equal(ck.keyswitch_key.lwe.a, ks_as[i])
        cells['expand %d' % R] = dict(per_tenant_ms=st['median_ms'] / R, range_ms=[st['min_ms'] / R, st['max_ms'] / R],
                                     decompress_per_tenant_ms=sd['median_ms'] / len(check),
                                     decompress_range_ms=[sd['min_ms'] / len(check), sd['max_ms'] / len(check)],
                                     identical=bool(ok))
        print('expand %d:' % R, cells['expand %d' % R], flush=True)
        del slots, ks_as
        gc.collect()
        torch.cuda.empty_cache()

    # --- T distinct tenants x 1 NAND, expansions every call
    xs, ys = samples(T, 1), samples(T, 1)
    results = {}
    for R in (128, 256):
        m = ctx.make_multi_key_machine(keys, resident_tenants=R)
        st, out = stats(lambda: m.gate_nand(xs, ys), args.reps)
        results[R] = out
        cells['nand %dx1 R=%d' % (T, R)] = dict(st, per_call_expansions=T)
        print('nand %dx1 R=%d:' % (T, R), st, flush=True)
        del m
        gc.collect()
        torch.cuda.empty_cache()
    ok = all(same(a, b) for a, b in zip(results[128], results[256]))
    for t in (0, 127, 128, T - 1):
        vm = ctx.make_virtual_machine(keys[t].decompress(thr))
        ok &= same(results[256][t], vm.gate_nand(xs[t], ys[t]))
        del vm
    cells['nand %dx1 R=128' % T]['identical'] = cells['nand %dx1 R=256' % T]['identical'] = bool(ok)
    del results, xs, ys
    gc.collect()
    torch.cuda.empty_cache()

    # --- 256 x 16 at R = 256 (second call: nothing to expand) against the resident machine on the same keys
    sub = keys[:256]
    del keys
    xs, ys = samples(256, 16), samples(256, 16)
    m = ctx.make_multi_key_machine(sub, resident_tenants=256)
    m.gate_nand(xs, ys)
    st, pooled = stats(lambda: m.gate_nand(xs, ys), args.reps)
    del m
    gc.collect()
    torch.cuda.empty_cache()
    resident = ctx.make_multi_key_machine([k.decompress(thr) for k in sub])
    sr, want = stats(lambda: resident.gate_nand(xs, ys), args.reps)
    ok = all(same(a, b) for a, b in zip(pooled, want))
    cells['256x16 R=256'] = dict(st, resident_median_ms=sr['median_ms'], resident_range_ms=[sr['min_ms'], sr['max_ms']],
                                 identical=bool(ok))
    print('256x16 R=256:', cells['256x16 R=256'], flush=True)

    res = dict(gpu=info, reps=args.reps, tenants=T, cells=cells)
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))
    assert all(c.get('identical', True) for c in cells.values()), 'outputs differ'


if __name__ == '__main__':
    main()
