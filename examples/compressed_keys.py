"""Compressed cloud keys and ciphertexts: the client generates keys and encrypts, and sends only seeds and bodies; the
server loads them, regenerates the masks on the GPU and computes a NAND gate; the client decrypts.

    python examples/compressed_keys.py
"""
import os
import sys

import numpy

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import nufhe_b200 as nufhe  # noqa: E402

# client: keys and compressed ciphertexts (SecureRNG: seeds and noises from os.urandom)
client = nufhe.Context(rng=nufhe.SecureRNG())
secret_key = client.make_secret_key()
cloud_key_bytes = client.make_cloud_key(secret_key, compressed=True).dumps()
size = 1024
rng = numpy.random.RandomState()
x, y = rng.randint(0, 2, size).astype(bool), rng.randint(0, 2, size).astype(bool)
x_bytes = client.encrypt(secret_key, x, compressed=True).dumps()
y_bytes = client.encrypt(secret_key, y, compressed=True).dumps()
print('cloud key: %d bytes compressed' % len(cloud_key_bytes))
print('ciphertexts: %d + %d bytes compressed for %d bits each' % (len(x_bytes), len(y_bytes), size))

# server: load, decompress on the GPU, compute
server = nufhe.Context()
cloud_key = server.load_compressed_cloud_key(cloud_key_bytes).decompress(server.thread)
vm = server.make_virtual_machine(cloud_key)
cx = server.load_compressed_ciphertext(x_bytes).decompress(server.thread)
cy = server.load_compressed_ciphertext(y_bytes).decompress(server.thread)
result_bytes = vm.gate_nand(cx, cy).dumps()
print('decompressed cloud key: %d bytes; result: %d bytes (results are ordinary ciphertexts)'
      % (len(cloud_key.dumps()), len(result_bytes)))

# client: decrypt
result = client.decrypt(secret_key, client.load_ciphertext(result_bytes))
assert (result == ~(x & y)).all()
print('NAND of %d encrypted bit pairs decrypts correctly' % size)
