"""The PRESENT block cipher's 4-bit S-box on 4096 encrypted nibbles, each held as two 2-bit digits, with tree-based
lookup tables (nufhe_b200/tree_lut.py): one table of two functions (the high and the low output digit) of two input
digits, three bootstraps per nibble on the GPU.  Checks every result and prints the time."""
import os
import sys
import time

import numpy
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import nufhe_b200   # noqa: E402

SBOX = numpy.array([0xC, 0x5, 0x6, 0xB, 0x9, 0x0, 0xA, 0xD, 0x3, 0xE, 0xF, 0x8, 0x4, 0x7, 0x1, 0x2])


def main():
    ctx = nufhe_b200.Context()
    sk = ctx.make_secret_key()
    cloud_key, tree_key = ctx.make_cloud_key(sk, tree_key=True)
    vm = ctx.make_virtual_machine(cloud_key)

    nibbles = numpy.random.RandomState(0).randint(0, 16, size=4096)
    hi, lo = ctx.encrypt_int(sk, nibbles >> 2, 2), ctx.encrypt_int(sk, nibbles & 3, 2)
    # tables[f, x_hi, x_lo]: f = 0 the high output digit, f = 1 the low one
    x = numpy.arange(16).reshape(4, 4)
    sbox = vm.make_tree_lut(numpy.stack([SBOX[x] >> 2, SBOX[x] & 3]), bits=2, digits=2)

    vm.lut_tree(tree_key, sbox, [hi, lo])                 # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out_hi, out_lo = vm.lut_tree(tree_key, sbox, [hi, lo])
    torch.cuda.synchronize()
    elapsed = time.perf_counter() - t0

    got = ctx.decrypt_int(sk, out_hi, 2) * 4 + ctx.decrypt_int(sk, out_lo, 2)
    assert (got == SBOX[nibbles]).all(), 'wrong S-box outputs'
    print('PRESENT S-box on %d encrypted nibbles: all correct, %.1f ms (%.0f nibbles/s) on %s'
          % (nibbles.size, elapsed * 1e3, nibbles.size / elapsed, torch.cuda.get_device_name(0)))


if __name__ == '__main__':
    main()
