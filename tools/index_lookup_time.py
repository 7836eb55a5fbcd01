"""Time encrypted-index lookups (DESIGN.md section 15) on one GPU: each entry point and whole vm.lookup calls at 4096
queries for m = 8, 12, 16, 20 (one column), and lut_tree at D = 4, P = 2 (an 8-bit table) for comparison.  CUDA events,
median of --reps calls after --warmup.  The selectors are random rows (the work does not depend on their values), so
the run needs no client-side encryption.  Prints one JSON object with the card name and power limit."""
import argparse
import json
import os
import subprocess
import sys

import numpy
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import nufhe_b200 as nufhe                      # noqa: E402
from nufhe_b200 import index_lookup as IL       # noqa: E402

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
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:            # (the figures are reported without a card line rather than not at all)
        out = 'unknown (%s)' % e
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--queries', type=int, default=4096)
    ap.add_argument('--bits', type=int, nargs='*', default=[8, 12, 16, 20])
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--no-tree', action='store_true')
    ap.add_argument('--out', help='also write the JSON object to this file')
    args = ap.parse_args()
    ctx = nufhe.Context(rng=nufhe.DeterministicRNG(1))
    sk = ctx.make_secret_key()
    ck, tk, ik = ctx.make_cloud_key(sk, tree_key=True, index_key=True)
    vm = ctx.make_virtual_machine(ck)
    thr = ctx.thread
    Q = args.queries
    res = {'card': card(), 'queries': Q, 'lookup': {}}
    for m in args.bits:
        sel = torch.randint(-2**31, 2**31, (Q, m, 2, 2, 2, N), dtype=torch.int32, device=thr.device)
        index = nufhe.EncryptedIndexArray(sk.params, m, sel, 0.0)
        table = vm.make_index_table(numpy.random.RandomState(m).randint(0, 4, size=1 << m), out='int', bits=2)
        r = {'queries_per_pass': IL.queries_per_pass(m, 1)}
        step = min(Q, r['queries_per_pass'])
        part = sel[:step]
        r['prepare_ms'] = median_ms(lambda: thr.index_prepare(part), args.warmup, args.reps)
        spec = thr.index_prepare(part).reshape(step, m, -1)
        levels = []
        cur = table.polys
        for j in range(10, m):
            nxt = thr.index_cmux_level(cur, spec, j, step)
            levels.append(median_ms(lambda c=cur, jj=j: thr.index_cmux_level(c, spec, jj, step), args.warmup, args.reps))
            cur = nxt
        r['cmux_levels_ms'] = levels
        r['rotate_extract_ms'] = median_ms(lambda: thr.index_rotate_extract(cur, spec, m, 1, step), args.warmup, args.reps)
        r['pass_queries'] = step
        del spec, cur
        r['lookup_ms'] = median_ms(lambda: vm.lookup(index, table), args.warmup, args.reps)
        r['external_products_per_query'] = (2**(m - 10) - 1 if m > 10 else 0) + min(m, 10)
        r['products_per_s'] = Q * r['external_products_per_query'] / (r['lookup_ms'] * 1e-3)
        # bytes the rotation streams: one 128 KB selector row per product
        r['rotate_key_gb_per_s'] = step * min(m, 10) * 16 * 512 * 16 / (r['rotate_extract_ms'] * 1e-3) / 1e9
        res['lookup'][m] = r
        del sel, index
        torch.cuda.empty_cache()
        print(json.dumps({m: r}), flush=True)
    if not args.no_tree:
        tab = numpy.random.RandomState(3).randint(0, 4, size=(4,) * 4)
        tree = vm.make_tree_lut(tab, 2, 4)
        digits = [ctx.encrypt_int(sk, numpy.random.RandomState(d).randint(0, 4, size=Q), 2) for d in range(4)]
        res['lut_tree_d4_p2_ms'] = median_ms(lambda: vm.lut_tree(tk, tree, digits), 1, 3)
    print(json.dumps(res))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
