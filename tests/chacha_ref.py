"""An independent ChaCha20 keystream in vectorised NumPy: the reference the seeded masks (csrc/chacha.cuh,
nb_seeded_uniform_i32) are checked against.  TEST INFRASTRUCTURE ONLY; it shares no code with the CUDA source.

The stream (DESIGN.md section 10): RFC 8439's block function with 20 rounds in the original 64-bit-counter state layout
-- words 0-3 the constants, 4-11 the seed, 12-13 the block counter (low word first), 14-15 the nonce (low word first).
Word i of the stream is word i % 16 of block i / 16."""
import numpy

_CONSTANTS = (0x61707865, 0x3320646e, 0x79622d32, 0x6b206574)
_U32 = numpy.uint32


def _rotl(x, s):
    return (x << _U32(s)) | (x >> _U32(32 - s))


def chacha20_blocks(seed, nonce, counters):
    """(len(counters), 16) uint32: the blocks with the given 64-bit counters of the stream (seed, nonce)."""
    seed = numpy.asarray(seed).astype(numpy.int64).astype(_U32).reshape(8)
    counters = numpy.asarray(counters, numpy.uint64).reshape(-1)
    nonce = int(nonce) & (2**64 - 1)
    nb = counters.size
    init = [numpy.full(nb, c, _U32) for c in _CONSTANTS]
    init += [numpy.full(nb, w, _U32) for w in seed]
    init += [(counters & numpy.uint64(0xffffffff)).astype(_U32), (counters >> numpy.uint64(32)).astype(_U32),
             numpy.full(nb, nonce & 0xffffffff, _U32), numpy.full(nb, nonce >> 32, _U32)]
    x = [v.copy() for v in init]

    def qr(a, b, c, d):
        x[a] += x[b]; x[d] ^= x[a]; x[d] = _rotl(x[d], 16)
        x[c] += x[d]; x[b] ^= x[c]; x[b] = _rotl(x[b], 12)
        x[a] += x[b]; x[d] ^= x[a]; x[d] = _rotl(x[d], 8)
        x[c] += x[d]; x[b] ^= x[c]; x[b] = _rotl(x[b], 7)

    for _ in range(10):
        qr(0, 4, 8, 12); qr(1, 5, 9, 13); qr(2, 6, 10, 14); qr(3, 7, 11, 15)
        qr(0, 5, 10, 15); qr(1, 6, 11, 12); qr(2, 7, 8, 13); qr(3, 4, 9, 14)
    return numpy.stack([x[i] + init[i] for i in range(16)], axis=1)


def chacha20_words(seed, nonce, first, count):
    """Words [first, first + count) of the stream (seed, nonce) as int32 (what nb_seeded_uniform_i32 writes)."""
    first, count = int(first), int(count)
    assert first >= 0 and count >= 0 and first + count <= 2**64
    if count == 0:
        return numpy.empty(0, numpy.int32)
    b0, b1 = first // 16, (first + count - 1) // 16
    blocks = chacha20_blocks(seed, nonce, numpy.arange(b1 - b0 + 1, dtype=numpy.uint64) + numpy.uint64(b0))
    return blocks.reshape(-1)[first % 16:first % 16 + count].view(numpy.int32)


def seeded_uniform(seed, nonce, shape, first=0):
    """Engine.seeded_uniform on the host: `shape` int32 values, stream words from `first` on in C order."""
    shape = tuple(shape)
    return chacha20_words(seed, nonce, first, int(numpy.prod(shape, dtype=numpy.int64))).reshape(shape)
