"""Many clients, each with its own keys, running a 2-digit tree lookup table and downloading packed results
(MultiKeyVirtualMachine.lut_tree and .pack, DESIGN.md section 18).  Each level of the tree LUT and each packing pass runs
once for all clients; every client's result is bit-identical to what a VirtualMachine with that client's keys alone
would return.

    python examples/multi_key_ops.py [clients]

Key generation dominates the run time of this example, so the clients share a few key sets (client t uses set t % 4);
a server would hold one set per client.
"""
import os
import sys

import numpy

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import nufhe_b200 as nufhe  # noqa: E402

ctx = nufhe.Context()
clients = int(sys.argv[1]) if len(sys.argv) > 1 else 256
sets = 4
rng = numpy.random.RandomState()

# each key set: secret key, cloud key, tree key (for lut_tree) and the packing key pair (for pack)
keys = []
for _ in range(sets):
    sk = ctx.make_secret_key()
    ck, tk = ctx.make_cloud_key(sk, tree_key=True)
    psk, pk = ctx.make_packing_keys(sk)
    keys.append((sk, ck, tk, psk, pk))

# f(hi, lo) on two 2-bit digits: the 4-bit number hi lo, reduced mod 3
table_values = (4 * numpy.arange(4)[:, None] + numpy.arange(4)[None, :]) % 3
vm = ctx.make_virtual_machine(keys[0][1])
table = vm.make_tree_lut(table_values, bits=2, digits=2)

# each client encrypts a few pairs of digits (client 3 is idle this time)
his, los, values = [], [], []
for t in range(clients):
    sk = keys[t % sets][0]
    if t == 3:
        his.append(None), los.append(None), values.append(None)
        continue
    hi, lo = rng.randint(0, 4, 1 + t % 5), rng.randint(0, 4, 1 + t % 5)
    his.append(ctx.encrypt_int(sk, hi, 2))
    los.append(ctx.encrypt_int(sk, lo, 2))
    values.append((hi, lo))

# the server: one machine for all cloud keys; two tree levels for everyone, then one packing pass for everyone
mk = ctx.make_multi_key_machine([keys[t % sets][1] for t in range(clients)])
tree_keys = [keys[t % sets][2] if values[t] is not None else None for t in range(clients)]
results = mk.lut_tree(tree_keys, table, [his, los])
packing_keys = [keys[t % sets][4] if values[t] is not None else None for t in range(clients)]
packed = mk.pack(packing_keys, results)

for t in range(clients):
    if values[t] is None:
        assert results[t] is None and packed[t] is None
        continue
    hi, lo = values[t]
    assert (ctx.decrypt_int(keys[t % sets][3], packed[t], 2) == table_values[hi, lo]).all()
print('a 2-digit tree LUT and packed results for %d clients with their own keys: all decrypt correctly' % clients)
