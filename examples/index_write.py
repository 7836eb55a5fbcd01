"""A private per-client counter array: clients increment counters at encrypted indexes, so that the server learns
neither which counter moved nor any count, then read the counts back by encrypted index (DESIGN.md section 21)."""
import os
import sys

import numpy

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import nufhe_b200 as nufhe   # noqa: E402

ctx = nufhe.Context()
sk = ctx.make_secret_key()
# the client keeps sk and index_key; the cloud key and tree key go to the server
cloud_key, tree_key, index_key = ctx.make_cloud_key(sk, tree_key=True, index_key=True)
vm = ctx.make_virtual_machine(cloud_key)

# 256 counters of 2 bits, starting at zero: the server needs no upload to start
m = 8
counters = vm.make_index_table(numpy.zeros(1 << m, int), bits=2)

# three rounds of increments at encrypted indexes (repeats add up); the server's work is the same for every index
rng = numpy.random.RandomState(0)
expected = numpy.zeros(1 << m, int)
for _ in range(3):
    hits = rng.randint(0, 1 << m, size=16)
    counters = vm.scatter_add(None, counters, ctx.encrypt_index(index_key, hits, m), 1)
    numpy.add.at(expected, hits, 1)
expected %= 4

# overwrite one counter with a value the server computed, at an index only the client knows
counters = vm.write(tree_key, counters, ctx.encrypt_index(index_key, [7], m), ctx.encrypt_int(sk, numpy.array([3]), 2))
expected[7] = 3

# read back every counter by encrypted index
got = ctx.decrypt_int(sk, vm.lookup(ctx.encrypt_index(index_key, numpy.arange(1 << m), m), counters), 2)
assert numpy.array_equal(got, expected)
print('48 private increments and one private overwrite of a 256-counter array: all counts read back correctly')
