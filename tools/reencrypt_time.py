"""Time re-encryption (DESIGN.md section 22) on one GPU at 1024, 4096 and 16 384 rows: nb_reencrypt alone against the
tree-key chain (nb_tree_keyswitch of the rotations X^(-p) C, then the coefficient-0 extraction) on the same inputs,
alternated call by call with the outputs compared, the recipient's key switch, and the whole vm.reencrypt; then
mk.reencrypt with 64 tenants of 64 rows each, and the device bytes per key of both routes.  CUDA events, median of
--reps calls after --warmup.  Prints one JSON object with the card's name, power limit and SM clocks, read in the same
run."""
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
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = 'unavailable: %s' % e
    return out


def rotations(sample, n):
    """The tree key of the rotations X^(-p) C, p < 2 n: masks (n, 2, 1, N) and bodies (n, 2, N) on the device."""
    j = torch.arange(N, device=sample.device)
    rows = []
    for p in range(2 * n):
        idx = (j + p) % N
        sign = torch.where(j + p < N, 1, -1).to(torch.int64)
        rows.append(sample.to(torch.int64)[:, idx] * sign)
    rot = torch.stack(rows)                                      # (2 n, 2, N)
    rot = ((rot & 0xffffffff) ^ (1 << 31)) - (1 << 31)
    rot = rot.to(torch.int32)
    return rot[:, 0].reshape(n, 2, 1, N).contiguous(), rot[:, 1].reshape(n, 2, N).contiguous()


def chain_output(V, b):
    """(0, b) minus the coefficient-0 extraction of V (R, 2, N)."""
    out_a = torch.cat([-V[:, 0, :1], V[:, 0, 1:].flip(1)], dim=1)
    return out_a, b - V[:, 1, 0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--rows', type=int, nargs='+', default=[1024, 4096, 16384])
    args = ap.parse_args()
    info = card()
    ctx = nufhe.Context(rng=nufhe.DeterministicRNG(2211))
    thr = ctx.thread
    skA = ctx.make_secret_key()
    skB = ctx.make_secret_key()
    ckB, cpkB = ctx.make_cloud_key(skB, compact_public_key=True)
    vm = ctx.make_virtual_machine(ckB)
    rekey = ctx.make_reencryption_key(skA, cpkB)
    n = rekey.n
    spec, body = rekey.spectra(thr)
    masks, bodies = rotations(rekey.sample.to(thr.device), n)
    planes = thr.tree_prepare(masks, bodies)
    ks = ckB.keyswitch_key.device_arrays()
    res = dict(card=info, warmup=args.warmup, reps=args.reps, rows={})
    for R in args.rows:
        bits = numpy.random.RandomState(R).randint(0, 2, size=R).astype(bool)
        ct = ctx.encrypt(skA, bits)
        fused = lambda: thr.reencrypt(ct.a, ct.b, [spec], [body], [R])
        chain = lambda: chain_output(thr.tree_keyswitch(ct.a, planes, 1), ct.b)
        fa, fb = fused()
        ca, cb = chain()
        equal = bool(torch.equal(fa, ca) and torch.equal(fb, cb))
        for f in (fused, chain):                                   # warm-up of both shapes
            for _ in range(args.warmup):
                f()
        tf, tc = [], []
        for _ in range(args.reps):                                 # alternated call by call
            tf.append(median_ms(fused, 0, 1))
            tc.append(median_ms(chain, 0, 1))
        keyswitch = median_ms(lambda: thr.keyswitch(ks, (fa, fb)), args.warmup, args.reps)
        whole = median_ms(lambda: vm.reencrypt(rekey, ct), args.warmup, args.reps)
        assert (ctx.decrypt(skB, vm.reencrypt(rekey, ct)) == bits).all()
        res['rows'][R] = dict(reencrypt_ms=float(numpy.median(tf)), tree_chain_ms=float(numpy.median(tc)),
                              outputs_equal=equal, keyswitch_ms=keyswitch, vm_reencrypt_ms=whole)
        print(R, res['rows'][R], flush=True)
    # 64 tenants of 64 rows
    T, rows = 64, 64
    cks, cpks = [], []
    for _ in range(T):
        sk = ctx.make_secret_key()
        ck, cpk = ctx.make_cloud_key(sk, compact_public_key=True)
        cks.append(ck), cpks.append(cpk)
    mk = ctx.make_multi_key_machine(cks)
    rekeys = [ctx.make_reencryption_key(skA, cpk) for cpk in cpks]
    cts = [ctx.encrypt(skA, numpy.ones(rows, bool)) for _ in range(T)]
    res['multikey'] = dict(tenants=T, rows_per_tenant=rows,
                           mk_reencrypt_ms=median_ms(lambda: mk.reencrypt(rekeys, cts), args.warmup, args.reps))
    res['bytes_per_key'] = dict(fused=spec.numel() * 8 + body.numel() * 4, tree_chain=planes.numel())
    print(json.dumps(res))


if __name__ == '__main__':
    main()
