"""Re-encryption: client A moves bits and 2-bit integers to client B on the server, without decrypting them and without
B's secret key.  A makes an 8 KB re-encryption key from B's published compact public key; the server re-encrypts A's
ciphertexts to B, combines them with B's own bits in a NAND gate and runs a LUT on the integers, and B decrypts
(DESIGN.md section 22)."""
import os
import sys

import numpy

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import nufhe_b200 as nufhe   # noqa: E402

ctx = nufhe.Context()

# client B: secret key, cloud key (given to the server) and the published compact public key
sk_b = ctx.make_secret_key()
cloud_b, compact_b = ctx.make_cloud_key(sk_b, compact_public_key=True)

# client A: encrypts its data under its own key, and makes the re-encryption key to B from B's public key alone.  The
# server must never give that key to B: with it and B's secret key, B would recover A's secret key.
sk_a = ctx.make_secret_key()
rng = numpy.random.RandomState(0)
bits_a = rng.randint(0, 2, 4096).astype(bool)
ints_a = rng.randint(0, 4, 4096)
ct_bits, ct_ints = ctx.encrypt(sk_a, bits_a), ctx.encrypt_int(sk_a, ints_a, 2)
rekey = ctx.load_reencryption_key(ctx.make_reencryption_key(sk_a, ctx.load_compact_public_key(compact_b.dumps())).dumps())

# the server, with B's cloud key: re-encrypt, then compute with B's own data
vm = ctx.make_virtual_machine(cloud_b)
bits_b = rng.randint(0, 2, 4096).astype(bool)
nand = vm.gate_nand(vm.reencrypt(rekey, ct_bits), ctx.encrypt(sk_b, bits_b))
table = numpy.array([0, 3, 1, 2])
mapped = vm.lut(vm.make_lut(table, 2), vm.reencrypt(rekey, ct_ints))

# client B decrypts
assert numpy.array_equal(ctx.decrypt(sk_b, nand), ~(bits_a & bits_b))
assert numpy.array_equal(ctx.decrypt_int(sk_b, mapped, 2), table[ints_a])
print('re-encryption key %d bytes: 4096 NANDs and 4096 LUTs on re-encrypted data correct' % len(rekey.dumps()))
