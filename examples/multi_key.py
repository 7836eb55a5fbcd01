"""Several clients, each with its own keys, and one server that evaluates all their gates in one fused launch
(MultiKeyVirtualMachine, DESIGN.md section 17).  Every client's result is bit-identical to what a VirtualMachine with
that client's cloud key alone would return.

    python examples/multi_key.py
"""
import os
import sys

import numpy

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import nufhe_b200 as nufhe  # noqa: E402

ctx = nufhe.Context()
clients = 8
rng = numpy.random.RandomState()

# each client: its own key pair and a few encrypted bits (client 5 has nothing to compute this time)
secret_keys, cloud_keys, xs, ys, bits = [], [], [], [], []
for t in range(clients):
    sk, ck = ctx.make_key_pair()
    secret_keys.append(sk)
    cloud_keys.append(ck)
    if t == 5:
        xs.append(None), ys.append(None), bits.append(None)
        continue
    x, y = rng.randint(0, 2, t + 1).astype(bool), rng.randint(0, 2, t + 1).astype(bool)
    xs.append(ctx.encrypt(sk, x))
    ys.append(ctx.encrypt(sk, y))
    bits.append((x, y))

# the server: one machine for all the cloud keys; one bootstrap launch and one key switch for every client's NAND
mk = ctx.make_multi_key_machine(cloud_keys)
results = mk.gate_nand(xs, ys)

# and one lookup table for everyone: x + y as a 2-bit integer
table = ctx.make_virtual_machine(cloud_keys[0]).make_lut([0, 1, 2, 3], bits=2)
ints = [None if b is None else ctx.encrypt_int(secret_keys[t], b[0].astype(int) + b[1], 2) for t, b in enumerate(bits)]
sums = mk.lut(table, ints)

for t in range(clients):
    if bits[t] is None:
        assert results[t] is None and sums[t] is None
        continue
    x, y = bits[t]
    assert (ctx.decrypt(secret_keys[t], results[t]) == ~(x & y)).all()
    assert (ctx.decrypt_int(secret_keys[t], sums[t], 2) == x.astype(int) + y).all()
print('NAND and a LUT for %d clients with their own keys, in one launch each: all decrypt correctly' % clients)
