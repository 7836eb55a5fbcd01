"""Packed results: the server packs gate outputs into GLWE samples, so the client downloads 4 bytes per bit instead of
about 2 KB.  Encrypt, run a gate, pack, pickle, load and decrypt, and print the sizes.

    python examples/packed_results.py
"""
import os
import sys

import numpy

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import nufhe_b200 as nufhe   # noqa: E402


def main(size=4096):
    ctx = nufhe.Context()
    secret_key, cloud_key = ctx.make_key_pair()
    # the client keeps packing_secret_key next to secret_key and sends packing_key to the server with the cloud key
    packing_secret_key, packing_key = ctx.make_packing_keys(secret_key)

    rng = numpy.random.RandomState(0)
    x, y = rng.randint(0, 2, (2, size)).astype(bool)
    cx, cy = ctx.encrypt(secret_key, x), ctx.encrypt(secret_key, y)

    vm = ctx.make_virtual_machine(cloud_key)
    result = vm.gate_nand(cx, cy)
    packed = vm.pack(packing_key, result)

    plain = result.dumps()
    wire = packed.dumps()
    back = ctx.load_packed_ciphertext(wire)
    bits = ctx.decrypt(packing_secret_key, back)
    assert (bits == ~(x & y)).all()
    print('%d NAND results: %.1f KB as LweSampleArray, %.1f KB packed (%.2f bytes per bit)'
          % (size, len(plain) / 1e3, len(wire) / 1e3, len(wire) / size))
    print('packing key: %.1f MB pickled' % (len(packing_key.dumps()) / 1e6))


if __name__ == '__main__':
    main()
