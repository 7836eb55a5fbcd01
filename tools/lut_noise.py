#!/usr/bin/env python
"""Measure the noise that decides which lookup-table configurations are safe (nufhe_b200/lut.py: check_noise), and the
throughput of lookup tables against gate_nand.

For each (L, shift) the tool makes 65 536 inputs that are themselves LUT outputs (fresh encryptions through an
identity table), forms the input the kernel rounds (x, or x * 2^shift + y), and computes on the host, with the secret
key, the phase the blind rotation actually uses: barb - sum bara_i s_i mod 2N with every term rounded to a multiple
of 2^L.  Its distance to the exact message position, in torus units, is the error whose standard deviation the
check compares with the box half-width 2^-(P + 2).  Throughput: LUT evaluations per second at B = 4096 for
L = 0, 1, 2 (bootstrap and key switch), and gate_nand at the same batch, timed with CUDA events.

    python tools/lut_noise.py [--evals 65536] [--out results.json]
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
from nufhe_b200 import lut  # noqa: E402

N = 1024


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True).stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0)


def rounded_phase_error(x, key, L, ideal_t32):
    """Torus-unit error of the mod-switched phase (rounded to multiples of 2^L) against the exact message."""
    a = x.a.cpu().numpy().astype(numpy.int64)
    b = x.b.cpu().numpy().astype(numpy.int64)

    def ms(v):
        return ((((v & 0xffffffff) + (1 << (20 + L))) & 0xffffffff) >> (21 + L)) << L
    p = (ms(b) - ms(a) @ key.astype(numpy.int64)) % (2 * N)
    ideal = (ideal_t32.astype(numpy.int64) & 0xffffffff) * (2 * N) / 2**32
    d = (p - ideal + N) % (2 * N) - N
    return d / (2 * N)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--evals', type=int, default=65536)
    ap.add_argument('--out', default=None, help='also write the results as JSON to this file')
    args = ap.parse_args()
    ctx = nufhe_b200.Context(rng=nufhe_b200.DeterministicRNG(2026))
    sk, ck = ctx.make_key_pair()
    vm = ctx.make_virtual_machine(ck)
    thr = ctx.thread
    key = sk.lwe_key.key.cpu().numpy()
    params = ck.params
    rng = numpy.random.RandomState(1)
    bits = 2                       # the error does not depend on P; P = 2 holds both bivariate packings below
    ident = vm.make_lut(list(range(2**bits)), bits)
    res = {'card': card(), 'evals': args.evals, 'sigma': []}
    for L in (0, 1, 2):
        for shift in (None, 0, 1):
            mx = rng.randint(0, 2, args.evals)
            x = vm.lut(ident, ctx.encrypt_int(sk, mx, bits))
            if shift is None:
                inp, m = x, mx
            else:
                my = rng.randint(0, 2, args.evals)
                y = vm.lut(ident, ctx.encrypt_int(sk, my, bits))
                inp = vm.empty_ciphertext(x.shape)
                thr.lwe_affine((inp.a, inp.b), (x.a, x.b), (y.a, y.b), 0, 1 << shift, 1)
                m = mx * 2**shift + my
            err = rounded_phase_error(inp, key, L, lut.encode_int(m, bits))
            est = lut._sigma_estimate(params.in_out_params, params.tgsw_params, params.ks_decomp_length,
                                      params.ks_log2_base, L, shift)
            row = {'L': L, 'shift': shift, 'sigma_measured': float(err.std()), 'sigma_estimate': est,
                   'mean': float(err.mean()), 'max_abs': float(numpy.abs(err).max())}
            res['sigma'].append(row)
            print(json.dumps(row), flush=True)

    # throughput at B = 4096: LUT (bootstrap + key switch) for L = 0, 1, 2 against gate_nand
    B, reps = 4096, 10
    x = ctx.encrypt_int(sk, rng.randint(0, 2, B), 1)
    bx = ctx.encrypt(sk, rng.randint(0, 2, B).astype(bool))
    tables = {0: vm.make_lut([1, 0], 1), 1: vm.make_lut([[1, 0], [0, 1]], 1), 2: vm.make_lut([[1, 0]] * 4, 1)}
    runs = {'gate_nand': lambda: vm.gate_nand(bx, bx)}
    for L, t in tables.items():
        runs['lut_L%d' % L] = (lambda t=t: vm.lut(t, x))
    res['throughput'] = {}
    for name, fn in runs.items():
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        outs = B << int(name[-1]) if name.startswith('lut') else B
        res['throughput'][name] = {'ms_per_call': ms, 'bootstraps_per_s': B / ms * 1e3, 'outputs_per_s': outs / ms * 1e3}
        print(name, json.dumps(res['throughput'][name]), flush=True)
    print('card:', res['card'])
    if args.out is None:
        return
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
        json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
