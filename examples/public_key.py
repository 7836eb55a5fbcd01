"""Public-key encryption: the key owner publishes a 66 KB public key; a third party holding only that key encrypts two
4096-bit vectors and a vector of 2-bit integers; the server computes a NAND gate and a lookup table; the owner decrypts.

    python examples/public_key.py
"""
import os
import sys

import numpy

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import nufhe_b200 as nufhe  # noqa: E402

# owner: secret key, cloud key for the server, public key for everyone
owner = nufhe.Context(rng=nufhe.SecureRNG())
secret_key = owner.make_secret_key()
cloud_key_bytes = owner.make_cloud_key(secret_key).dumps()
public_key_bytes = owner.make_public_key(secret_key).dumps()
print('public key: %d bytes' % len(public_key_bytes))

# sender: only the public key; it can encrypt but not decrypt
size = 4096
sender = nufhe.Context(rng=nufhe.SecureRNG())
public_key = sender.load_public_key(public_key_bytes)
rng = numpy.random.RandomState()
x, y = rng.randint(0, 2, size).astype(bool), rng.randint(0, 2, size).astype(bool)
v = rng.randint(0, 4, size)
x_bytes, y_bytes = sender.encrypt(public_key, x).dumps(), sender.encrypt(public_key, y).dumps()
v_bytes = sender.encrypt_int(public_key, v, 2).dumps()

# server: NAND of the bits, v -> v^2 mod 4 on the integers
server = nufhe.Context()
vm = server.make_virtual_machine(server.load_cloud_key(cloud_key_bytes))
nand_bytes = vm.gate_nand(server.load_ciphertext(x_bytes), server.load_ciphertext(y_bytes)).dumps()
square_bytes = vm.lut(vm.make_lut([0, 1, 0, 1], 2), server.load_ciphertext(v_bytes)).dumps()

# owner: decrypt
assert (owner.decrypt(secret_key, owner.load_ciphertext(nand_bytes)) == ~(x & y)).all()
assert (owner.decrypt_int(secret_key, owner.load_ciphertext(square_bytes), 2) == v * v % 4).all()
print('NAND of %d bit pairs and a LUT on %d 2-bit integers, encrypted with the public key, decrypt correctly'
      % (size, size))
