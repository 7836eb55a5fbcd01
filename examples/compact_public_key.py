"""Compact public-key encryption: a third party that holds only a 5 KB compact public key encrypts 4096 bits in 16 KB
(4 bytes per bit); the server expands them into ordinary ciphertexts, evaluates NAND and packs the results, which the
key holder downloads at 4 bytes per bit and decrypts (DESIGN.md sections 16 and 12)."""
import os
import sys

import numpy

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import nufhe_b200 as nufhe   # noqa: E402

# the key holder: secret key, cloud key and compact public key, and a packing key pair for the download
ctx = nufhe.Context()
sk = ctx.make_secret_key()
cloud_key, compact_pk = ctx.make_cloud_key(sk, compact_public_key=True)
packing_sk, packing_key = ctx.make_packing_keys(sk)
published = compact_pk.dumps()

# a third party (a sensor, another service) encrypts its readings with the published key alone
sender = nufhe.Context(rng=nufhe.SecureRNG(), thread=ctx.thread)
rng = numpy.random.RandomState(0)
x, y = rng.randint(0, 2, (2, 4096)).astype(bool)
pk = sender.load_compact_public_key(published)
upload = [sender.encrypt(pk, x).dumps(), sender.encrypt(pk, y).dumps()]

# the server expands the uploads, computes and packs
vm = ctx.make_virtual_machine(cloud_key)
cx, cy = (vm.expand(ctx.load_compact_ciphertext(u)) for u in upload)
download = vm.pack(packing_key, vm.gate_nand(cx, cy)).dumps()

# the key holder decrypts
got = ctx.decrypt(packing_sk, ctx.load_packed_ciphertext(download))
assert numpy.array_equal(got, ~(x & y))
print('public key %d bytes, upload %d bytes per 4096 bits, download %d bytes: NAND of 4096 bit pairs correct'
      % (len(published), len(upload[0]), len(download)))
