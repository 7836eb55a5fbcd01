"""Encrypted-index table lookups: 4096 private queries into a table of 2^16 two-bit entries.  The client encrypts its
indices bit by bit (TGSW selectors); the server looks them up with CMux gates only, without learning which entries
were read, and the results are ordinary ciphertexts that feed gates and LUTs (DESIGN.md section 15)."""
import os
import sys

import numpy

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import nufhe_b200 as nufhe   # noqa: E402

ctx = nufhe.Context()
sk = ctx.make_secret_key()
cloud_key, index_key = ctx.make_cloud_key(sk, index_key=True)      # the client keeps sk and index_key
vm = ctx.make_virtual_machine(cloud_key)

rng = numpy.random.RandomState(0)
table = rng.randint(0, 4, size=1 << 16)                            # the server's data
queries = rng.randint(0, 1 << 16, size=4096)                       # the client's indices

index = ctx.encrypt_index(index_key, queries, 16)                  # 16 selectors per query
result = vm.lookup(index, vm.make_index_table(table, out='int', bits=2))
got = ctx.decrypt_int(sk, result, 2)
assert numpy.array_equal(got, table[queries])

# the results are ordinary ciphertexts: "is the entry nonzero" as a gate bit, then NAND with a fresh bit
nonzero = vm.make_lut([0, 1, 1, 1], 2, out='bool')
bits = rng.randint(0, 2, size=4096).astype(bool)
out = vm.gate_nand(vm.lut(nonzero, result), ctx.encrypt(sk, bits))
assert numpy.array_equal(ctx.decrypt(sk, out), ~((table[queries] != 0) & bits))
print('4096 lookups into a 2^16-entry table: all correct, and NAND of the results correct')
