"""A cloud key with a multi-bit bootstrap key: key bits taken two at a time (DESIGN.md section 14).  Gates, lookup
tables and their results work as with the default key; the key is opt-in because it is slower on an H100 today and
carries more noise (section 14 has the measurements)."""
import os
import sys

import numpy

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import nufhe_b200 as nufhe  # noqa: E402


def main():
    ctx = nufhe.Context()
    sk = ctx.make_secret_key()
    ck = ctx.make_cloud_key(sk, multi_bit=2)
    print(type(ck.bootstrap_key).__name__, 'with', ck.bootstrap_key.tgsw.shape[0], 'TGSW rows')
    vm = ctx.make_virtual_machine(ck)
    rng = numpy.random.RandomState(0)
    a, b = rng.randint(0, 2, 4096).astype(bool), rng.randint(0, 2, 4096).astype(bool)
    r = vm.gate_nand(ctx.encrypt(sk, a), ctx.encrypt(sk, b))
    assert (ctx.decrypt(sk, r) == ~(a & b)).all()
    x = rng.randint(0, 4, 4096)
    inc = vm.make_lut([1, 2, 3, 0], 2)
    assert (ctx.decrypt_int(sk, vm.lut(inc, ctx.encrypt_int(sk, x, 2)), 2) == (x + 1) % 4).all()
    print('4096 NAND gates and 4096 lookups with a multi-bit key: ok')


if __name__ == '__main__':
    main()
