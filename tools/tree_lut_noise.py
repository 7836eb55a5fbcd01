#!/usr/bin/env python
"""Measure the noise of tree-based LUT outputs (nufhe_b200/tree_lut.py: tree_sigma, MEASURED_SIGMA), as
tools/lut_noise.py does for one-level LUTs.

For each (P, D) the tool evaluates an identity-like table on --evals fresh digit encryptions (f = the lowest digit, so
every path of the tree is taken), and computes on the host, with the secret key, the mod-switched phase that a
following one-input LUT would use: barb - sum bara_i s_i mod 2N.  Its distance to the exact message position, in
torus units, is the error whose standard deviation tree_lut compares with the box half-width 2^-(P + 2).  Also prints
the sample standard deviation of the unrounded output phase against tree_lut.output_variance.

    python tools/tree_lut_noise.py [--evals 65536] [--out results.json]
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
from lut_noise import card, rounded_phase_error  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--evals', type=int, default=65536)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    print('card:', card())
    ctx = nufhe_b200.Context(rng=nufhe_b200.DeterministicRNG(2027))
    sk = ctx.make_secret_key()
    ck, tk = ctx.make_cloud_key(sk, tree_key=True)
    vm = ctx.make_virtual_machine(ck)
    key = sk.lwe_key.key.cpu().numpy()
    rng = numpy.random.RandomState(3)
    res = {'card': card(), 'evals': args.evals, 'sigma': {}, 'estimate': {}, 'phase_sigma': {}, 'phase_estimate': {}}
    for bits, D in ((2, 2), (2, 3), (2, 4), (1, 2), (1, 3), (1, 4)):
        M = 1 << bits
        table = numpy.broadcast_to(numpy.arange(M), (M,) * D)          # f = d_0
        values = [rng.randint(0, M, args.evals) for _ in range(D)]
        out = vm.lut_tree(tk, vm.make_tree_lut(table, bits, D), [ctx.encrypt_int(sk, v, bits) for v in values])
        ideal = lut.encode_int(values[-1], bits)
        err = rounded_phase_error(out, key, 0, ideal)
        a, b = out.a.cpu().numpy().astype(numpy.int64), out.b.cpu().numpy().astype(numpy.int64)
        ph = ((b - a @ key.astype(numpy.int64) - ideal.astype(numpy.int64) + 2**31) % 2**32 - 2**31) / 2**32
        name = 'P%d_D%d' % (bits, D)
        res['sigma'][name] = float(err.std())
        res['estimate'][name] = float(tree_lut.tree_sigma(sk.params, bits, D))
        res['phase_sigma'][name] = float(ph.std())
        res['phase_estimate'][name] = float(tree_lut.output_variance(sk.params, bits, D)**0.5)
        print(name, 'rounded-phase sigma %.5f (estimate %.5f), margin %.1f; output phase sigma %.5f (estimate %.5f)'
              % (err.std(), res['estimate'][name], 2.0**-(bits + 2) / err.std(), ph.std(), res['phase_estimate'][name]))
    print(json.dumps(res))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
