"""Time lookups into encrypted tables against plaintext tables (DESIGN.md section 20) on one GPU, in the same process:
vm.lookup at 4096 queries for m = 8, 12, 16, 20 (one column) into an IndexTable and into an EncryptedIndexTable made
with the compact public key, the two calls alternated rep by rep; then vm.make_encrypted_table from 2^16 gate outputs.
CUDA events, median of --reps calls after --warmup.  The selectors are random rows (the work does not depend on their
values).  Prints one JSON object with the card name, power limit and maximum SM clock."""
import argparse
import json
import os
import subprocess
import sys

import numpy
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import nufhe_b200 as nufhe                      # noqa: E402

N = 1024


def timed_ms(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e)


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
    ap.add_argument('--build-entries', type=int, default=1 << 16)
    ap.add_argument('--out', help='also write the JSON object to this file')
    args = ap.parse_args()
    ctx = nufhe.Context(rng=nufhe.DeterministicRNG(1))
    sk = ctx.make_secret_key()
    ck, tk, cpk = ctx.make_cloud_key(sk, tree_key=True, compact_public_key=True)
    vm = ctx.make_virtual_machine(ck)
    thr = ctx.thread
    Q = args.queries
    res = {'card': card(), 'queries': Q, 'lookup': {}}
    for m in args.bits:
        sel = torch.randint(-2**31, 2**31, (Q, m, 2, 2, 2, N), dtype=torch.int32, device=thr.device)
        index = nufhe.EncryptedIndexArray(sk.params, m, sel, 0.0)
        raw = numpy.random.RandomState(m).randint(0, 4, size=1 << m)
        tables = {'plain': vm.make_index_table(raw, out='int', bits=2), 'encrypted': ctx.encrypt_table(cpk, raw, bits=2)}
        for t in tables.values():
            for _ in range(args.warmup):
                vm.lookup(index, t)
        times = {k: [] for k in tables}
        for _ in range(args.reps):
            for k, t in tables.items():
                times[k].append(timed_ms(lambda: vm.lookup(index, t)))
        r = {k + '_ms': float(numpy.median(v)) for k, v in times.items()}
        r['ratio'] = r['encrypted_ms'] / r['plain_ms']
        res['lookup'][m] = r
        del sel, index, tables
        torch.cuda.empty_cache()
        print(json.dumps({m: r}), flush=True)
    B = args.build_entries
    bits = numpy.random.RandomState(2).randint(0, 2, size=(2, B)).astype(bool)
    col = vm.gate_nand(ctx.encrypt(sk, bits[0]), ctx.encrypt(sk, bits[1]))
    for _ in range(args.warmup):
        vm.make_encrypted_table(tk, col, out='bool')
    res['build_entries'] = B
    res['build_ms'] = float(numpy.median([timed_ms(lambda: vm.make_encrypted_table(tk, col, out='bool'))
                                          for _ in range(args.reps)]))
    print(json.dumps(res))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
