"""Time oblivious writes (DESIGN.md section 21) beside lookups of the same table on one GPU, in the same process: the
device work of a scatter_add of --queries LWE values (tree key switch, assembly, rotation, demultiplexer, accumulation
and 16-bit rounding) and vm.lookup of as many indexes into one encrypted table, for m = 8, 16, 20, the two alternated
rep by rep; then the same with one table per tenant (16 tenants) against mk.lookup.  The write runs below the noise
rule of vm.scatter_add, which refuses 4096 queries in one call (every query adds noise to every entry): the work, and
so the time, of a call does not depend on that rule.  CUDA events, median of --reps calls after --warmup.  Selectors
and values are random (the work does not depend on them).  Prints one JSON object with the card name, power limit and
maximum SM clock."""
import argparse
import json
import os
import sys

import numpy
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import nufhe_b200 as nufhe                      # noqa: E402
from nufhe_b200 import index_lookup as IL       # noqa: E402
from nufhe_b200 import index_write              # noqa: E402
from nufhe_b200.batch_keys import OneKey, TenantKeys     # noqa: E402
from encrypted_table_time import card, timed_ms  # noqa: E402


def random_index(ctx, params, m, q, rng):
    rows = rng.randint(-2**31, 2**31, size=(q, m, 2, 2, 2, IL.N), dtype=numpy.int64).astype(numpy.int32)
    return IL.EncryptedIndexArray(params, m, ctx.thread.to_device(rows), 0.0)


def random_values(ctx, params, q, rng):
    n = params.in_out_params.size
    a = rng.randint(-2**31, 2**31, size=(q, 1, n), dtype=numpy.int64).astype(numpy.int32)
    b = rng.randint(-2**31, 2**31, size=(q, 1), dtype=numpy.int64).astype(numpy.int32)
    return ctx.thread.to_device(a), ctx.thread.to_device(b)


def write_work(thr, params, keys, tables, sels, a, b, ids=None):
    """The device work of one scatter_add call into `tables` (one per tenant, or one)."""
    m = tables[0].bits
    accs = torch.stack([index_write.table_nodes(t) for t in tables])
    index_write.scatter_passes(thr, params, keys, m, 1, sels, a, b, accs, ids)
    return IL._round16(accs)


def median_pair(f, g, warmup, reps):
    for _ in range(warmup):
        f(), g()
    tf, tg = [], []
    for _ in range(reps):
        tf.append(timed_ms(f))
        tg.append(timed_ms(g))
    return float(numpy.median(tf)), float(numpy.median(tg))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--bits', type=int, nargs='+', default=[8, 16, 20])
    ap.add_argument('--queries', type=int, default=4096)
    ap.add_argument('--tenants', type=int, default=16)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--reps', type=int, default=5)
    args = ap.parse_args()
    ctx = nufhe.Context(rng=nufhe.DeterministicRNG(1))
    sk = ctx.make_secret_key()
    ck, tk, ik = ctx.make_cloud_key(sk, tree_key=True, index_key=True)
    vm = ctx.make_virtual_machine(ck)
    params = sk.params
    rng = numpy.random.RandomState(0)
    out = {'card': card(), 'queries': args.queries, 'single_key': {}, 'multi_key': {}}
    for m in args.bits:
        t = ctx.encrypt_table(ik, numpy.zeros(1 << m, int), bits=2)
        index = random_index(ctx, params, m, args.queries, rng)
        a, b = random_values(ctx, params, args.queries, rng)
        sels = [index.samples.reshape(args.queries, m, 2, 2, 2, IL.N)]
        w, r = median_pair(lambda: write_work(ctx.thread, params, OneKey(ctx.thread, tree_key=tk), [t], sels, a, b),
                           lambda: vm.lookup(index, t), args.warmup, args.reps)
        out['single_key'][m] = {'scatter_add_ms': w, 'lookup_ms': r}
        print(json.dumps({'m': m, 'scatter_add_ms': w, 'lookup_ms': r}), file=sys.stderr)
    T, per = args.tenants, args.queries // args.tenants
    keys = [ctx.make_cloud_key(s, tree_key=True, index_key=True) for s in [ctx.make_secret_key() for _ in range(T)]]
    machine = ctx.make_multi_key_machine([k[0] for k in keys])
    for m in args.bits:
        tables = [ctx.encrypt_table(k[2], numpy.zeros(1 << m, int), bits=2) for k in keys]
        idx = [random_index(ctx, params, m, per, rng) for _ in range(T)]
        a, b = random_values(ctx, params, per * T, rng)
        sels = [x.samples.reshape(per, m, 2, 2, 2, IL.N) for x in idx]
        tkeys = TenantKeys(ctx.thread, [per] * T, planes=[k[1].planes(ctx.thread) for k in keys])
        ids = numpy.repeat(numpy.arange(T, dtype=numpy.uint32), per)
        w, r = median_pair(lambda: write_work(ctx.thread, params, tkeys, tables, sels, a, b, ids),
                           lambda: machine.lookup(idx, tables), args.warmup, args.reps)
        out['multi_key'][m] = {'tenants': T, 'scatter_add_ms': w, 'lookup_ms': r}
        print(json.dumps({'m': m, 'tenants': T, 'scatter_add_ms': w, 'lookup_ms': r}), file=sys.stderr)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
