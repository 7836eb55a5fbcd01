"""NumPy restatement of the tensor-core key switch (kernels.cuh: keyswitch_mma_kernel, ks_prepare_kernel).

res = -OneHot . Key mod 2^32, as one u8 x u8 -> s32 GEMM over the 4 byte planes of the key: K runs over the 24 576
(j, k, d >= 1) rows in the kernel's stage order, N over 512 padded columns (ks_a, ks_b in column 500) in 4 planes."""
import numpy

IN, T, N_OUT, GROUPS = 1024, 8, 500, 256


def k_order():
    """(j, k, d) of every K index: stage G, then kpos < 96 as ks_mma_k_index splits it"""
    G, kpos = numpy.meshgrid(numpy.arange(GROUPS), numpy.arange(96), indexing='ij')
    c, h, tig, e = kpos >> 5, (kpos >> 4) & 1, (kpos >> 2) & 3, kpos & 3
    return (G + GROUPS * tig).ravel(), (4 * h + 3 - e).ravel(), (c + 1).ravel()


def digits(src_a):
    """(B, 1024, 8) base-4 digits of the rounded input coefficients, k = 0 most significant"""
    v = (src_a.astype(numpy.uint32) + numpy.uint32(1 << 15)) >> numpy.uint32(16)
    return (v[..., None] >> (14 - 2 * numpy.arange(T, dtype=numpy.uint32))) & 3


def key_matrix(ks_a, ks_b):
    """(24576, 512) uint32 key rows in K order: ks_a, then ks_b, then zero columns"""
    j, k, d = k_order()
    m = numpy.zeros((j.size, 512), numpy.uint32)
    m[:, :N_OUT] = ks_a[j, k, d].view(numpy.uint32)
    m[:, N_OUT] = ks_b[j, k, d].view(numpy.uint32)
    return m


def keyswitch(ks_a, ks_b, src_a, src_b):
    """(res_a, res_b) int32 via the GEMM: one-hot rows, exact plane sums, recombination mod 2^32"""
    j, k, d = k_order()
    one_hot = (digits(src_a)[:, j, k] == d).astype(numpy.int64)                    # (B, 24576)
    key = key_matrix(ks_a, ks_b)
    total = numpy.zeros((src_a.shape[0], 512), numpy.uint64)
    for p in range(4):
        s = one_hot @ ((key >> numpy.uint32(8 * p)) & 0xFF).astype(numpy.int64)    # exact: < 8192 * 255 < 2^21
        assert s.max(initial=0) < 2**21
        total += s.astype(numpy.uint64) << numpy.uint64(8 * p)
    total = (numpy.uint64(0) - total) & numpy.uint64(0xFFFFFFFF)
    res = total.astype(numpy.uint32)
    res_b = (src_b.astype(numpy.uint32) + res[:, N_OUT]).view(numpy.int32)
    return res[:, :N_OUT].view(numpy.int32), res_b
