#!/usr/bin/env python
"""Measure the noise that decides which configurations a multi-bit bootstrap key allows (DESIGN.md section 14;
nufhe_b200/lut.py: MEASURED_SIGMA_MULTI_BIT, nufhe_b200/tree_lut.py: MEASURED_SIGMA_MULTI_BIT), as tools/lut_noise.py
and tools/tree_lut_noise.py do for the standard key.  Every bootstrap here uses a multi-bit cloud key.

* LUTs: for each (L, shift), --evals inputs that are themselves LUT outputs (fresh encryptions through an identity
  table), the input the kernel rounds (x, or x * 2^shift + y), and the error of its mod-switched phase (every term
  rounded to a multiple of 2^L) against the exact message position, in torus units.
* gate_nand: the same error for the input of a NAND whose two inputs are NAND outputs, against the box half-width 1/8.
* Trees: the error of the mod-switched phase of a level-D output, for (P, D) up to one level past what the estimate
  allows (the noise rule is bypassed for the measurement only).

    python tools/multibit_noise.py [--evals 65536] [--out results.json]
"""
import argparse
import json
import os
import sys

import numpy

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import nufhe_b200  # noqa: E402
from nufhe_b200 import lut, tree_lut  # noqa: E402
from nufhe_b200.gates import MU  # noqa: E402
from lut_noise import card, rounded_phase_error  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--evals', type=int, default=65536)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    res = {'card_before': card(), 'evals': args.evals, 'lut': [], 'tree': [], 'gate_nand': None}
    print('card:', res['card_before'], flush=True)
    ctx = nufhe_b200.Context(rng=nufhe_b200.DeterministicRNG(2028))
    sk = ctx.make_secret_key()
    ck, tk = ctx.make_cloud_key(sk, tree_key=True, multi_bit=2)
    vm = ctx.make_virtual_machine(ck)
    thr = ctx.thread
    key = sk.lwe_key.key.cpu().numpy()
    params = ck.params
    rng = numpy.random.RandomState(1)

    bits = 2                       # the error does not depend on P; P = 2 holds both bivariate packings below
    ident = vm.make_lut(list(range(2**bits)), bits)
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
                                      params.ks_log2_base, L, shift, multi_bit=2)
            row = {'L': L, 'shift': shift, 'sigma_measured': float(err.std()), 'sigma_estimate': est,
                   'mean': float(err.mean()), 'max_abs': float(numpy.abs(err).max())}
            res['lut'].append(row)
            print(json.dumps(row), flush=True)

    # gate_nand: inputs that are NAND outputs, the prologue (0, 1/8) - a - b rounded to [0, 2N)
    a, b, c, d = (rng.randint(0, 2, args.evals).astype(bool) for _ in range(4))
    u = vm.gate_nand(ctx.encrypt(sk, a), ctx.encrypt(sk, b))
    v = vm.gate_nand(ctx.encrypt(sk, c), ctx.encrypt(sk, d))
    inp = vm.empty_ciphertext(u.shape)
    thr.lwe_affine((inp.a, inp.b), (u.a, u.b), (v.a, v.b), 1 << 29, -1, -1)
    mu_u = numpy.where(~(a & b), int(MU), -int(MU)).astype(numpy.int64)
    mu_v = numpy.where(~(c & d), int(MU), -int(MU)).astype(numpy.int64)
    ideal = ((2**29 - mu_u - mu_v) & 0xffffffff).astype(numpy.uint32).view(numpy.int32)
    err = rounded_phase_error(inp, key, 0, ideal)
    est = (2 * lut.bootstrap_variance(params, 2) + (params.in_out_params.size / 2 + 1) / 2048**2 / 12)**0.5
    res['gate_nand'] = {'sigma_measured': float(err.std()), 'sigma_estimate': est, 'margin_sigmas': 0.125 / float(err.std()),
                        'max_abs': float(numpy.abs(err).max())}
    print('gate_nand', json.dumps(res['gate_nand']), flush=True)

    # trees: the rule is bypassed so that one level past the estimate's limit can be measured
    tree_lut._check_config = lambda *a, **k: None
    for P, D in ((2, 2), (2, 3), (1, 2), (1, 3), (1, 4)):
        M = 1 << P
        table = numpy.broadcast_to(numpy.arange(M), (M,) * D)          # f = d_0
        values = [rng.randint(0, M, args.evals) for _ in range(D)]
        out = vm.lut_tree(tk, vm.make_tree_lut(table, P, D), [ctx.encrypt_int(sk, v, P) for v in values])
        err = rounded_phase_error(out, key, 0, lut.encode_int(values[-1], P))
        row = {'P': P, 'D': D, 'sigma_measured': float(err.std()),
               'sigma_estimate': float(tree_lut.tree_sigma(params, P, D, multi_bit=2)),
               'margin_sigmas': 2.0**-(P + 2) / float(err.std()), 'max_abs': float(numpy.abs(err).max())}
        res['tree'].append(row)
        print(json.dumps(row), flush=True)
    res['card_after'] = card()
    print('card:', res['card_after'])
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
