#!/usr/bin/env python
"""Time the multi-key tree LUT, packing, expansion, index lookup and per-tenant-table LUT (DESIGN.md section 18)
against a loop over per-tenant VirtualMachines issuing the same calls, alternated in one process, with CUDA events.

    python tools/multikey_ops_time.py [--keys 8] [--reps 3] [--mixes 2048x1,256x16,16x256] [--ops ...] [--json PATH]

Tenant t uses key t % K of K distinct key sets (cloud key, tree key, packing key, compact public key, index key), and
its VirtualMachine is that key's.  The operations: a 2-digit tree LUT on 2-bit digits (one function), packing of the
tenant's ciphertexts, expansion of its compact ciphertexts, a lookup of 8-bit indices in a one-column table and a
one-output LUT with the tenant's own table.  Both sides' outputs are compared bit for bit.  The card's name, power
limit and SM clock limit are read in the same run.  Prints one line per (mix, operation) and one JSON object at the end.
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

OPS = ('lut_tree', 'pack', 'expand', 'lookup', 'lut')


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
    fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end)


def flat(x):
    """The tensors of a result, in a fixed order, for a bitwise comparison."""
    if x is None:
        return []
    if isinstance(x, (list, tuple)):
        return [v for y in x for v in flat(y)]
    if hasattr(x, 'data') and x.data.dtype == torch.uint16:
        return [x.data.view(torch.int16)]
    return [x.a, x.b, x.current_variances]


def identical(xs, ys):
    fx, fy = flat(xs), flat(ys)
    return len(fx) == len(fy) and all(torch.equal(a, b) for a, b in zip(fx, fy))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--keys', type=int, default=8, help='distinct key sets the tenants cycle through')
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--mixes', default='2048x1,256x16,16x256')
    ap.add_argument('--ops', default=','.join(OPS))
    ap.add_argument('--json', default=None, help='also write the results to this file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('multikey_ops_time.py measures on a CUDA device; there is none')
    import nufhe_b200 as nufhe
    from nufhe_b200.index_lookup import EncryptedIndexArray

    ctx = nufhe.Context(rng=nufhe.DeterministicRNG(20261019))
    K = args.keys
    sks, cks, tks, iks, cpks, pks = [], [], [], [], [], []
    for _ in range(K):
        sk = ctx.make_secret_key()
        ck, tk, ik, cpk = ctx.make_cloud_key(sk, tree_key=True, index_key=True, compact_public_key=True)
        pk = ctx.make_packing_keys(sk)[1]
        for lst, v in zip((sks, cks, tks, iks, cpks, pks), (sk, ck, tk, ik, cpk, pk)):
            lst.append(v)
    vms = [ctx.make_virtual_machine(ck) for ck in cks]
    tree_table = vms[0].make_tree_lut(numpy.arange(16).reshape(4, 4) % 4, bits=2, digits=2)
    index_table = vms[0].make_index_table(numpy.arange(256) % 4, bits=2)
    luts = [vms[0].make_lut([(v + k) % 4 for v in range(4)], bits=2) for k in range(K)]
    torch.cuda.synchronize()
    info = gpu_info()
    print('device:', torch.cuda.get_device_name(0), '|', info, '| key sets:', K, flush=True)

    rng = numpy.random.RandomState(1)
    results = []
    for mix in args.mixes.split(','):
        T, per = (int(v) for v in mix.split('x'))
        machine = ctx.make_multi_key_machine([cks[t % K] for t in range(T)])
        tenants_of = [list(range(k, T, K)) for k in range(K)]

        def per_key(enc):
            """enc(k, (n_k, per) values) -> an array indexable by a tenant's position among key k's tenants."""
            out = [None] * T
            for k, ts in enumerate(tenants_of):
                if ts:
                    arr = enc(k, rng.randint(0, 4, size=(len(ts), per)))
                    for i, t in enumerate(ts):
                        out[t] = arr(i)
            return out
        d1 = per_key(lambda k, v: ctx.encrypt_int(sks[k], v, 2).__getitem__)
        d0 = per_key(lambda k, v: ctx.encrypt_int(sks[k], v, 2).__getitem__)

        def index(k, v):
            e = ctx.encrypt_index(iks[k], v, 8)
            return lambda i: EncryptedIndexArray(e.params, 8, e.samples[i], e.variance)
        idx = per_key(index)
        comp = [ctx.encrypt(cpks[t % K], rng.randint(0, 2, per).astype(bool)) for t in range(T)]
        ops = {
            'lut_tree': (lambda: machine.lut_tree([tks[t % K] for t in range(T)], tree_table, [d1, d0]),
                         lambda: [vms[t % K].lut_tree(tks[t % K], tree_table, [d1[t], d0[t]]) for t in range(T)]),
            'pack': (lambda: machine.pack([pks[t % K] for t in range(T)], d0),
                     lambda: [vms[t % K].pack(pks[t % K], d0[t]) for t in range(T)]),
            'expand': (lambda: machine.expand(comp), lambda: [vms[t % K].expand(comp[t]) for t in range(T)]),
            'lookup': (lambda: machine.lookup(idx, index_table),
                       lambda: [vms[t % K].lookup(idx[t], index_table) for t in range(T)]),
            'lut': (lambda: machine.lut([luts[t % K] for t in range(T)], d0),
                    lambda: [vms[t % K].lut(luts[t % K], d0[t]) for t in range(T)]),
        }
        for name in args.ops.split(','):
            multi, loop = ops[name]
            got, want = multi(), loop()                     # warm-up, and the outputs compared
            torch.cuda.synchronize()
            same = identical(got, want)
            del got, want
            t_mk, t_loop = [], []
            for _ in range(args.reps):                      # alternated
                t_mk.append(timed(multi))
                t_loop.append(timed(loop))
            med = lambda v: float(numpy.median(v))
            row = {'mix': mix, 'op': name, 'tenants': T, 'per_tenant': per, 'bit_identical': bool(same),
                   'multi_ms': med(t_mk), 'multi_ms_range': [min(t_mk), max(t_mk)],
                   'loop_ms': med(t_loop), 'loop_ms_range': [min(t_loop), max(t_loop)],
                   'speedup': med(t_loop) / med(t_mk)}
            results.append(row)
            print('%-8s %-8s multi %9.2f ms [%8.2f, %8.2f]  loop %9.2f ms [%8.2f, %8.2f]  x%6.2f  identical=%s' % (
                mix, name, row['multi_ms'], min(t_mk), max(t_mk), row['loop_ms'], min(t_loop), max(t_loop),
                row['speedup'], same), flush=True)
        del machine, d0, d1, idx, comp, ops
        torch.cuda.empty_cache()
    summary = {'device': torch.cuda.get_device_name(0), 'nvidia_smi': info, 'key_sets': K, 'reps': args.reps,
               'time': time.strftime('%Y-%m-%d %H:%M:%S'), 'results': results}
    print(json.dumps(summary))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(summary, f, indent=1)


if __name__ == '__main__':
    main()
