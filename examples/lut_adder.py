"""A 4-bit ripple-carry adder on encrypted integers with programmable bootstrapping: every bit position takes one
bootstrap with two outputs (sum and carry of a + b + carry, message space P = 2), where the gate version needs five
bootstraps per full adder."""
import os
import random
import sys
import time

import numpy

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import nufhe_b200 as nufhe   # noqa: E402

size, width, P = 4096, 4, 2
xs = numpy.array([random.randrange(16) for _ in range(size)])
ys = numpy.array([random.randrange(16) for _ in range(size)])

ctx = nufhe.Context()
secret_key, cloud_key = ctx.make_key_pair()
vm = ctx.make_virtual_machine(cloud_key)

# bit i of each operand, one ciphertext array per bit position, holding 0 or 1 in a 2-bit message space
a = [ctx.encrypt_int(secret_key, (xs >> i) & 1, P) for i in range(width)]
b = [ctx.encrypt_int(secret_key, (ys >> i) & 1, P) for i in range(width)]
# v = a + b + carry in [0, 3]: sum = v mod 2, carry = v >= 2, both from one blind rotation
full_adder = vm.make_lut([[v % 2 for v in range(4)], [v // 2 for v in range(4)]], P)


def add():
    out, carry = [], None
    for i in range(width):
        v = vm.int_add(a[i], b[i]) if carry is None else vm.int_add(vm.int_add(a[i], b[i]), carry)
        s, carry = vm.lut(full_adder, v)
        out.append(s)
    return out + [carry]


add()                                                   # warm-up
ctx.thread.synchronize()
t = time.time()
result = add()
ctx.thread.synchronize()
dt = time.time() - t

total = sum(ctx.decrypt_int(secret_key, r, P).astype(numpy.int64) << i for i, r in enumerate(result))
assert (total == xs + ys).all()
print('%d 4-bit additions in %.1f ms (%d two-output bootstraps of %d ciphertexts)' % (size, dt * 1e3, width, size))
