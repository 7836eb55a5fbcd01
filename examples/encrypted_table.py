"""A private record store: records stored encrypted on the server and read by encrypted index, so that the server
learns neither which record was read nor what any record holds (DESIGN.md section 20).  A second table is built on
the server from results it computed, and read the same way."""
import os
import sys

import numpy

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import nufhe_b200 as nufhe   # noqa: E402

ctx = nufhe.Context()
sk = ctx.make_secret_key()
# the client keeps sk and index_key; the cloud key, tree key and compact public key go to the server
cloud_key, tree_key, index_key, public_key = ctx.make_cloud_key(sk, tree_key=True, index_key=True,
                                                                compact_public_key=True)
vm = ctx.make_virtual_machine(cloud_key)

# 4096 records of two 2-bit fields, uploaded encrypted (whoever holds the compact public key may upload)
rng = numpy.random.RandomState(0)
records = rng.randint(0, 4, size=(2, 1 << 12))
store = ctx.load_encrypted_table(ctx.encrypt_table(public_key, records, bits=2).dumps())     # 32 KB on the wire

# private reads: 256 encrypted record numbers
wanted = rng.randint(0, 1 << 12, size=256)
field0, field1 = vm.lookup(ctx.encrypt_index(index_key, wanted, 12), store)
assert numpy.array_equal(ctx.decrypt_int(sk, field0, 2), records[0][wanted])
assert numpy.array_equal(ctx.decrypt_int(sk, field1, 2), records[1][wanted])

# a table of results the server computed (here the NAND of two encrypted bit vectors), read by encrypted index
a, b = rng.randint(0, 2, size=(2, 1 << 10)).astype(bool)
computed = vm.make_encrypted_table(tree_key, vm.gate_nand(ctx.encrypt(sk, a), ctx.encrypt(sk, b)), out='bool')
bits = vm.lookup(ctx.encrypt_index(index_key, wanted % 1024, 10), computed)
assert numpy.array_equal(ctx.decrypt(sk, bits), ~(a & b)[wanted % 1024])
print('256 private reads from an encrypted 4096-record store and from a server-built table: all correct')
