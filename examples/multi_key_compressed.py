"""A server with a few hundred clients that each upload a compressed cloud key (about 8.3 MB) and keeps only a few
dozen of them expanded on the GPU at a time (MultiKeyVirtualMachine with resident_tenants, DESIGN.md section 19).  A
gate for every client runs in rounds; every client's result is bit-identical to what a VirtualMachine with that
client's decompressed cloud key alone would return.

    python examples/multi_key_compressed.py
"""
import os
import sys

import numpy

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import nufhe_b200 as nufhe  # noqa: E402

ctx = nufhe.Context()
clients, resident = 300, 32
rng = numpy.random.RandomState()

# each client: its own secret key, a compressed cloud key sent to the server, and two encrypted bits
secret_keys, compressed_keys, xs, ys, bits = [], [], [], [], []
for t in range(clients):
    sk = ctx.make_secret_key()
    secret_keys.append(sk)
    compressed_keys.append(ctx.load_compressed_cloud_key(ctx.make_cloud_key(sk, compressed=True).dumps()))
    x, y = rng.randint(0, 2, 2).astype(bool), rng.randint(0, 2, 2).astype(bool)
    xs.append(ctx.encrypt(sk, x))
    ys.append(ctx.encrypt(sk, y))
    bits.append((x, y))

# the server: 300 compressed keys, at most 32 expanded (about 164 MB each) at any time
mk = ctx.make_multi_key_machine(compressed_keys, resident_tenants=resident)
results = mk.gate_nand(xs, ys)
print('after one NAND per client, the resident tenants are', mk.resident[:4], '...', mk.resident[-4:])

for t in range(clients):
    x, y = bits[t]
    assert (ctx.decrypt(secret_keys[t], results[t]) == ~(x & y)).all()
# a client's own machine on its decompressed key gives the same bits
vm = ctx.make_virtual_machine(compressed_keys[0].decompress(ctx.thread))
assert (vm.gate_nand(xs[0], ys[0]).a == results[0].a).all()
print('NAND for %d clients with %d resident keys: all results correct' % (clients, resident))
