"""Engine: one (CUDA device, stream) binding of the native library -- what a Reikna `Thread` is to the
reference (nufhe/api_high_level.py:153-181).  All methods take torch CUDA tensors (int32 for Torus32
data, int64 holding the uint64 bit patterns of field elements) and enqueue work on the engine's stream.
PyTorch is used for device memory and streams only.
"""
import ctypes
import weakref

import numpy
import torch

from . import _native

N = 1024


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


class Engine:

    def __init__(self, device=None, stream=None):
        if not torch.cuda.is_available():
            raise RuntimeError('nufhe_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback')
        self.lib = _native.load()
        if device is None:
            device = torch.cuda.current_device()
        self.device = torch.device('cuda', device if isinstance(device, int) else torch.device(device).index or 0)
        self.torch_stream = stream
        handle = ctypes.c_void_p()
        stream_ptr = ctypes.c_void_p(stream.cuda_stream if stream is not None else 0)
        rc = self.lib.nb_ctx_create(self.device.index, stream_ptr, ctypes.byref(handle))
        self.handle = handle
        self._stream_ptr = stream_ptr.value or 0
        self._ks_registrations = {}           # ks_a address -> token of its live ks_prepare registration
        if rc != _native.NB_OK:
            try:
                _native.check(handle, rc, 'nb_ctx_create')
            finally:
                if handle:
                    self.lib.nb_ctx_destroy(handle)
                self.handle = None
        self.device_params = DeviceParams(self.device)

    def __del__(self):
        h = getattr(self, 'handle', None)
        if h:
            self.lib.nb_ctx_destroy(h)
            self.handle = None

    # --- plumbing -------------------------------------------------------------------------
    def _call(self, name, *args):
        # work goes to torch's current stream on the engine's device unless the engine was given its own stream: that
        # is what keeps the native launches ordered with torch's copies / fills and lets torch.cuda.graph capture them
        if self.torch_stream is None:
            cur = torch.cuda.current_stream(self.device).cuda_stream
            if cur != self._stream_ptr:
                _native.check(self.handle, self.lib.nb_ctx_set_stream(self.handle, ctypes.c_void_p(cur)), 'nb_ctx_set_stream')
                self._stream_ptr = cur
        _native.check(self.handle, getattr(self.lib, name)(self.handle, *args), name)

    def reserve(self, batch):
        """Pre-allocate the native scratch for launches of up to `batch` ciphertexts (needed before graph capture)."""
        self._call('nb_ctx_reserve', int(batch))

    def synchronize(self):
        self._call('nb_ctx_synchronize')

    def build_info(self):
        return self.lib.nb_build_info().decode()

    def empty(self, shape, dtype):
        return torch.empty(tuple(shape), dtype=dtype, device=self.device)

    def to_device(self, arr):
        arr = numpy.ascontiguousarray(arr)
        if arr.dtype == numpy.uint64:
            arr = arr.view(numpy.int64)
        return torch.from_numpy(arr).to(self.device)

    @staticmethod
    def to_host(t, unsigned=False):
        arr = t.detach().cpu().numpy()
        return arr.view(numpy.uint64) if unsigned else arr

    def _dense(self, t, dtype):
        assert t.is_cuda and t.dtype == dtype, (t.device, t.dtype, dtype)
        return t if t.is_contiguous() else t.contiguous()

    # --- transforms -----------------------------------------------------------------------
    def ntt_forward_i32(self, x):
        x = self._dense(x, torch.int32)
        out = self.empty(x.shape, torch.int64)
        self._call('nb_ntt_forward_i32', _ptr(x), _ptr(out), x.numel() // N)
        return out

    def ntt_forward_u64(self, x):
        x = self._dense(x, torch.int64)
        out = self.empty(x.shape, torch.int64)
        self._call('nb_ntt_forward_u64', _ptr(x), _ptr(out), x.numel() // N)
        return out

    def ntt_inverse_i32(self, x):
        x = self._dense(x, torch.int64)
        out = self.empty(x.shape, torch.int32)
        self._call('nb_ntt_inverse_i32', _ptr(x), _ptr(out), x.numel() // N)
        return out

    def ntt_inverse_u64(self, x):
        x = self._dense(x, torch.int64)
        out = self.empty(x.shape, torch.int64)
        self._call('nb_ntt_inverse_u64', _ptr(x), _ptr(out), x.numel() // N)
        return out

    def ff_op(self, op, a, b=None):
        a = self._dense(a, torch.int64)
        out = torch.empty_like(a)
        period = 0
        if b is not None:
            b = self._dense(b, torch.int64)
            if b.numel() != a.numel():
                assert a.numel() % b.numel() == 0
                period = b.numel()
        self._call('nb_ff_elementwise', op, _ptr(a), _ptr(b), _ptr(out), a.numel(), period)
        return out

    # --- bootstrap path -------------------------------------------------------------------
    def bk_prepare(self, bk_ref):
        bk_ref = self._dense(bk_ref, torch.int64)
        rows = bk_ref.numel() // (8 * N)
        out = self.empty((rows, self.lib.nb_bk_row_u64()), torch.int64)
        self._call('nb_bk_prepare', _ptr(bk_ref), _ptr(out), rows)
        return out

    def bk_prepare_multibit(self, bk_ref):
        """A multi-bit bootstrap key (3 reference rows per group of two key bits) as the fused kernels read it: the FP64
        spectra of every row (nb_bk_prepare_multibit).  The result goes wherever a `bk_prepare` key goes."""
        bk_ref = self._dense(bk_ref, torch.int64)
        rows = bk_ref.numel() // (8 * N)
        if rows % 3:
            raise ValueError('a multi-bit key has 3 rows per group, got %d rows' % rows)
        out = self.empty((rows, self.lib.nb_bk_multibit_row_u64()), torch.int64)
        self._call('nb_bk_prepare_multibit', _ptr(bk_ref), _ptr(out), rows // 3)
        return out

    def external_product(self, accum, bk_int, row):
        """accum (B,2,1024) int32 is updated in place: accum <- bk[row] (x) accum"""
        assert accum.is_contiguous() and accum.dtype == torch.int32
        self._call('nb_external_product', _ptr(accum), _ptr(bk_int), row, accum.numel() // (2 * N))
        return accum

    def blind_rotate(self, accum, bara, bk_int, extract=True, return_accum=False):
        accum = self._dense(accum, torch.int32)
        bara = self._dense(bara, torch.int32)
        B = accum.numel() // (2 * N)
        n = bara.shape[-1]                    # (an empty batch is a no-op in the library)
        out_a = self.empty((B, N), torch.int32) if extract else None
        out_b = self.empty((B,), torch.int32) if extract else None
        acc_out = torch.empty_like(accum) if return_accum else None
        self._call('nb_blind_rotate', _ptr(accum), _ptr(bara), _ptr(bk_int), n, _ptr(out_a), _ptr(out_b),
                   _ptr(acc_out), B)
        return out_a, out_b, acc_out

    def bootstrap_extract(self, x1, x2, c, s1, s2, mu, bk_int, out=None):
        """x = (0,c) + s1*x1 + s2*x2 (x2 may be None); returns the extracted sample (a (B,1024), b (B,))."""
        a1, b1 = x1
        a1 = self._dense(a1, torch.int32)
        b1 = self._dense(b1, torch.int32)
        a2 = b2 = None
        if x2 is not None:
            a2 = self._dense(x2[0], torch.int32)
            b2 = self._dense(x2[1], torch.int32)
        B = b1.numel()
        n = a1.shape[-1]
        out_a, out_b = out if out is not None else (self.empty((B, N), torch.int32), self.empty((B,), torch.int32))
        self._call('nb_bootstrap_extract', _ptr(a1), _ptr(b1), _ptr(a2), _ptr(b2), int(c), int(s1), int(s2),
                   int(mu), _ptr(bk_int), n, _ptr(out_a), _ptr(out_b), B)
        return out_a, out_b

    def bootstrap_lut_extract(self, x1, x2, c, s1, s2, tv, log2_outputs, bk_int):
        """The programmable bootstrap of x = (0,c) + s1*x1 + s2*x2 (x2 may be None) with test vector `tv`: (1024,) int32
        for the whole batch or (B, 1024) for one per ciphertext.  Returns the 2^L extracted samples of every ciphertext,
        a (B * 2^L, 1024) and b (B * 2^L,), sample j of ciphertext c in row c * 2^L + j (nb_bootstrap_lut_extract)."""
        a1, b1 = self._dense(x1[0], torch.int32), self._dense(x1[1], torch.int32)
        a2 = b2 = None
        if x2 is not None:
            a2, b2 = self._dense(x2[0], torch.int32), self._dense(x2[1], torch.int32)
        tv = self._dense(tv, torch.int32)
        B = b1.numel()
        n = a1.shape[-1]
        stride = 0 if tv.dim() == 1 else N
        assert tv.shape[-1] == N and (stride == 0 or tv.numel() == B * N), (tuple(tv.shape), B)
        rows = B << int(log2_outputs)
        out_a, out_b = self.empty((rows, N), torch.int32), self.empty((rows,), torch.int32)
        self._call('nb_bootstrap_lut_extract', _ptr(a1), _ptr(b1), _ptr(a2), _ptr(b2), int(c), int(s1), int(s2),
                   _ptr(tv), stride, int(log2_outputs), _ptr(bk_int), n, _ptr(out_a), _ptr(out_b), B)
        return out_a, out_b

    def bootstrap_extract2(self, job_a, job_b, mu, bk_int):
        """Two bootstraps in one launch.  job = (x1, x2, c, s1, s2) as for bootstrap_extract.
        Returns two extracted samples (views of one (2B, 1024) / (2B,) allocation)."""
        def parts(job):
            x1, x2, c, s1, s2 = job
            a1, b1 = self._dense(x1[0], torch.int32), self._dense(x1[1], torch.int32)
            a2 = b2 = None
            if x2 is not None:
                a2, b2 = self._dense(x2[0], torch.int32), self._dense(x2[1], torch.int32)
            return a1, b1, a2, b2, int(c), int(s1), int(s2)
        pa, pb = parts(job_a), parts(job_b)
        B = pa[1].numel()
        n = pa[0].shape[-1]
        out_a, out_b = self.empty((2 * B, N), torch.int32), self.empty((2 * B,), torch.int32)
        self._call('nb_bootstrap_extract2', _ptr(pa[0]), _ptr(pa[1]), _ptr(pa[2]), _ptr(pa[3]), pa[4], pa[5], pa[6],
                   _ptr(pb[0]), _ptr(pb[1]), _ptr(pb[2]), _ptr(pb[3]), pb[4], pb[5], pb[6], int(mu), _ptr(bk_int), n,
                   _ptr(out_a), _ptr(out_b), B)
        return (out_a[:B], out_b[:B]), (out_a[B:], out_b[B:])

    def keyswitch(self, ks, src1, src2=None, c=0, out=None, want_cv=False):
        ks_a, ks_b, ks_cv = ks
        in_size, t, base, n = ks_a.shape
        a1 = self._dense(src1[0], torch.int32)
        b1 = self._dense(src1[1], torch.int32)
        a2 = b2 = None
        if src2 is not None:
            a2 = self._dense(src2[0], torch.int32)
            b2 = self._dense(src2[1], torch.int32)
        B = b1.numel()
        if out is None:
            res_a = self.empty(tuple(b1.shape) + (n,), torch.int32)
            res_b = self.empty(tuple(b1.shape), torch.int32)
        else:
            res_a, res_b = out
        res_cv = self.empty(tuple(b1.shape), torch.float32) if want_cv else None
        self._call('nb_keyswitch', _ptr(a1), _ptr(b1), _ptr(a2), _ptr(b2), int(c), _ptr(ks_a), _ptr(ks_b),
                   _ptr(ks_cv), in_size, n, t, int(base).bit_length() - 1, _ptr(res_a), _ptr(res_b),
                   _ptr(res_cv), B)
        return res_a, res_b, res_cv

    # --- multi-key calls (nb_mk_*, DESIGN.md section 17): tenant t owns counts[t] consecutive ciphertexts of the batch
    @staticmethod
    def _host_array(ctype, values):
        return (ctype * max(len(values), 1))(*values)

    def _mk_keys(self, bk_ints, counts):
        return (self._host_array(ctypes.c_void_p, [k.data_ptr() for k in bk_ints]),
                self._host_array(ctypes.c_size_t, [int(c) for c in counts]), len(bk_ints))

    def mk_bootstrap_extract(self, x1, x2, c, s1, s2, mu, bk_ints, counts):
        """bootstrap_extract over the ciphertexts of several keys: bk_ints[t] (bk_prepare) serves the counts[t]
        ciphertexts of tenant t, which follow those of tenant t - 1 (nb_mk_bootstrap_extract)."""
        a1, b1 = self._dense(x1[0], torch.int32), self._dense(x1[1], torch.int32)
        a2 = b2 = None
        if x2 is not None:
            a2, b2 = self._dense(x2[0], torch.int32), self._dense(x2[1], torch.int32)
        B = b1.numel()
        out_a, out_b = self.empty((B, N), torch.int32), self.empty((B,), torch.int32)
        keys, cnt, T = self._mk_keys(bk_ints, counts)
        self._call('nb_mk_bootstrap_extract', _ptr(a1), _ptr(b1), _ptr(a2), _ptr(b2), int(c), int(s1), int(s2),
                   int(mu), keys, cnt, T, a1.shape[-1], _ptr(out_a), _ptr(out_b), B)
        return out_a, out_b

    def mk_bootstrap_lut_extract(self, x1, x2, c, s1, s2, tv, log2_outputs, bk_ints, counts):
        """bootstrap_lut_extract over the ciphertexts of several keys, split as for mk_bootstrap_extract
        (nb_mk_bootstrap_lut_extract); tv (1024,) serves the whole batch, tv (B, 1024) holds one per ciphertext."""
        a1, b1 = self._dense(x1[0], torch.int32), self._dense(x1[1], torch.int32)
        a2 = b2 = None
        if x2 is not None:
            a2, b2 = self._dense(x2[0], torch.int32), self._dense(x2[1], torch.int32)
        tv = self._dense(tv, torch.int32)
        B = b1.numel()
        stride = 0 if tv.dim() == 1 else N
        assert tuple(tv.shape) == ((N,) if stride == 0 else (B, N)), (tuple(tv.shape), B)
        rows = B << int(log2_outputs)
        out_a, out_b = self.empty((rows, N), torch.int32), self.empty((rows,), torch.int32)
        keys, cnt, T = self._mk_keys(bk_ints, counts)
        self._call('nb_mk_bootstrap_lut_extract', _ptr(a1), _ptr(b1), _ptr(a2), _ptr(b2), int(c), int(s1), int(s2),
                   _ptr(tv), stride, int(log2_outputs), keys, cnt, T, a1.shape[-1], _ptr(out_a), _ptr(out_b), B)
        return out_a, out_b

    def mk_bootstrap_glwe_lut_extract(self, x, tv, bk_ints, counts):
        """bootstrap_glwe_lut_extract over the ciphertexts of several keys, split as for mk_bootstrap_extract
        (nb_mk_bootstrap_glwe_lut_extract)."""
        a, b = self._dense(x[0], torch.int32), self._dense(x[1], torch.int32)
        tv = self._dense(tv, torch.int32)
        B = b.numel()
        n = a.shape[-1]
        if tuple(tv.shape) != (B, 2, N) or a.numel() != B * n:
            raise ValueError('mk_bootstrap_glwe_lut_extract: tv %s for %d ciphertexts' % (tuple(tv.shape), B))
        out_a, out_b = self.empty((B, N), torch.int32), self.empty((B,), torch.int32)
        keys, cnt, T = self._mk_keys(bk_ints, counts)
        self._call('nb_mk_bootstrap_glwe_lut_extract', _ptr(a), _ptr(b), _ptr(tv), keys, cnt, T, n, _ptr(out_a),
                   _ptr(out_b), B)
        return out_a, out_b

    def mk_tree_keyswitch(self, a, planes, counts, mask_size):
        """tree_keyswitch over the rows of several tenants: planes[t] (tree_prepare) serves the counts[t] rows of tenant
        t (nb_mk_tree_keyswitch).  Returns V (R, k+1, N)."""
        a = self._dense(a, torch.int32)
        rows, n = a.shape
        want = self.lib.nb_tree_planes_bytes(n, int(mask_size))
        for t, p in enumerate(planes):
            if p.numel() != want:
                raise ValueError('mk_tree_keyswitch: tenant %d: %d plane bytes do not fit n = %d, k = %d'
                                 % (t, p.numel(), n, mask_size))
        out = self.empty((rows, mask_size + 1, N), torch.int32)
        self._call('nb_mk_tree_keyswitch', _ptr(a), self._host_array(ctypes.c_void_p, [p.data_ptr() for p in planes]),
                   self._host_array(ctypes.c_size_t, [int(c) for c in counts]), len(planes), n, int(mask_size),
                   _ptr(out), rows)
        return out

    def mk_ntt_mac(self, x, keys, group_counts):
        """ntt_mac over the groups of several tenants: keys[t] (R, U, N) serves the group_counts[t] groups of tenant t
        (nb_mk_ntt_mac).  Returns (G, U, N)."""
        x = self._dense(x, torch.int64)
        keys = [self._dense(k, torch.int64) for k in keys]
        if x.dim() != 3 or x.shape[2] != N or not keys or any(tuple(k.shape) != tuple(keys[0].shape) for k in keys) \
                or keys[0].dim() != 3 or keys[0].shape[2] != N or x.shape[1] != keys[0].shape[0]:
            raise ValueError('mk_ntt_mac: x %s and keys %s are not (G, R, N) and (R, U, N)'
                             % (tuple(x.shape), [tuple(k.shape) for k in keys]))
        groups, rows = x.shape[:2]
        outs = keys[0].shape[1]
        out = self.empty((groups, outs, N), torch.int64)
        self._call('nb_mk_ntt_mac', _ptr(x), self._host_array(ctypes.c_void_p, [k.data_ptr() for k in keys]),
                   self._host_array(ctypes.c_size_t, [int(c) for c in group_counts]), len(keys), _ptr(out), rows, outs,
                   groups)
        return out

    def mk_bootstrap_extract2(self, job_a, job_b, mu, bk_ints, counts):
        """bootstrap_extract2 over the ciphertexts of several keys: both jobs are split by the same counts
        (nb_mk_bootstrap_extract2).  Returns the two samples as views of one allocation."""
        def parts(job):
            x1, x2, c, s1, s2 = job
            a1, b1 = self._dense(x1[0], torch.int32), self._dense(x1[1], torch.int32)
            a2 = b2 = None
            if x2 is not None:
                a2, b2 = self._dense(x2[0], torch.int32), self._dense(x2[1], torch.int32)
            return a1, b1, a2, b2, int(c), int(s1), int(s2)
        pa, pb = parts(job_a), parts(job_b)
        B = pa[1].numel()
        out_a, out_b = self.empty((2 * B, N), torch.int32), self.empty((2 * B,), torch.int32)
        keys, cnt, T = self._mk_keys(bk_ints, counts)
        self._call('nb_mk_bootstrap_extract2', _ptr(pa[0]), _ptr(pa[1]), _ptr(pa[2]), _ptr(pa[3]), pa[4], pa[5], pa[6],
                   _ptr(pb[0]), _ptr(pb[1]), _ptr(pb[2]), _ptr(pb[3]), pb[4], pb[5], pb[6], int(mu), keys, cnt, T,
                   pa[0].shape[-1], _ptr(out_a), _ptr(out_b), B)
        return (out_a[:B], out_b[:B]), (out_a[B:], out_b[B:])

    def mk_keyswitch(self, keys, counts, src1, src2=None, c=0, want_cv=False):
        """keyswitch over the ciphertexts of several keys: keys[t] = (ks_a, ks_b, ks_cv) of tenant t serves its counts[t]
        rows (nb_mk_keyswitch).  Returns res_a (B, n), res_b (B,) and the variances (B,) or None."""
        in_size, t, base, n = keys[0][0].shape if keys else (0, 0, 0, 0)
        a1, b1 = self._dense(src1[0], torch.int32), self._dense(src1[1], torch.int32)
        a2 = b2 = None
        if src2 is not None:
            a2, b2 = self._dense(src2[0], torch.int32), self._dense(src2[1], torch.int32)
        B = b1.numel()
        res_a, res_b = self.empty((B, n), torch.int32), self.empty((B,), torch.int32)
        res_cv = self.empty((B,), torch.float32) if want_cv else None
        ks = [self._host_array(ctypes.c_void_p, [k[i].data_ptr() for k in keys]) for i in range(3)]
        self._call('nb_mk_keyswitch', _ptr(a1), _ptr(b1), _ptr(a2), _ptr(b2), int(c), ks[0], ks[1], ks[2],
                   self._host_array(ctypes.c_size_t, [int(x) for x in counts]), len(keys), in_size, n, t,
                   int(base).bit_length() - 1, _ptr(res_a), _ptr(res_b), _ptr(res_cv), B)
        return res_a, res_b, res_cv

    # --- expansion of compressed cloud keys into multi-key slots (DESIGN.md section 19)
    def mk_bk_slot(self, n):
        """An uninitialised slot for the bootstrap key of one tenant: n engine key rows (nb_bk_row_u64() words each).
        Its registration on this engine, which mk_bk_expand makes, is dropped when the slot is freed
        (nb_mk_slot_release), so that memory the allocator hands out again never passes for a key."""
        slot = self.empty((n, self.lib.nb_bk_row_u64()), torch.int64)
        weakref.finalize(slot, self._mk_slot_release, slot.data_ptr())
        return slot

    def _mk_slot_release(self, ptr):
        if self.handle:
            self.lib.nb_mk_slot_release(self.handle, ctypes.c_void_p(ptr))

    @staticmethod
    def _seeds(seeds):
        seeds = numpy.ascontiguousarray(numpy.asarray(seeds).astype(numpy.int64).astype(numpy.uint32).reshape(-1, 8))
        return seeds, seeds.ctypes.data_as(ctypes.c_void_p)

    def mk_bk_expand(self, seeds, bodies, slots, params):
        """The FP64 part of the engine key of every listed tenant into its slot (mk_bk_slot), in one launch
        (nb_mk_bk_expand): seeds (T, 8) of the compressed keys, bodies[t] (n, k+1, l, N) int32 on this device; the slots'
        contents equal bk_prepare of the decompressed key's FP64 part, word for word."""
        seeds, seeds_p = self._seeds(seeds)
        bodies = [self._dense(b, torch.int32) for b in bodies]
        n = params.in_out_params.size
        for b, s in zip(bodies, slots):
            assert b.shape[0] == n and s.is_contiguous() and s.shape == (n, self.lib.nb_bk_row_u64()), (b.shape, s.shape)
        tl = params.tgsw_params.tlwe_params
        self._call('nb_mk_bk_expand', seeds_p, self._host_array(ctypes.c_void_p, [b.data_ptr() for b in bodies]),
                   self._host_array(ctypes.c_void_p, [s.data_ptr() for s in slots]), len(slots), n, tl.mask_size,
                   params.tgsw_params.decomp_length, tl.polynomial_degree)

    def mk_ks_expand(self, seeds, ks_as):
        """The masks of every listed tenant's key-switch key into its ks_a (in, t, base, n) int32, rows h = 0 zero, in
        one launch (nb_mk_ks_expand): byte-identical to CompressedCloudKey.decompress()'s ks_a."""
        seeds, seeds_p = self._seeds(seeds)
        if not ks_as:
            return
        in_size, t, base, n = ks_as[0].shape
        assert all(k.is_contiguous() and k.shape == ks_as[0].shape for k in ks_as)
        self._call('nb_mk_ks_expand', seeds_p, self._host_array(ctypes.c_void_p, [k.data_ptr() for k in ks_as]),
                   len(ks_as), in_size, t, int(base).bit_length() - 1, n)

    def ks_prepare(self, ks_a, ks_b):
        """Lay a key-switch key (in = 1024, n = 500, t = 8, base 4) into the byte planes of the tensor-core key switch
        and register them for (ks_a, ks_b) on this engine (nb_ks_prepare).  Returns the planes, which must stay alive
        while the registration is wanted, or None when the key's d = 0 rows are not zero: such a key keeps the gather
        kernel.  The registration is dropped when the planes, ks_a or ks_b are freed, so that a later key at the same
        addresses never meets these planes.  Preparing the key again moves its registration to the new planes.
        Prepare outside any captured region: it allocates and synchronizes."""
        assert ks_a.is_contiguous() and ks_b.is_contiguous()
        in_size, t, base, n = ks_a.shape
        planes = self.empty((self.lib.nb_ks_prepared_bytes(),), torch.uint8)
        registered = ctypes.c_int(0)
        self._call('nb_ks_prepare', _ptr(ks_a), _ptr(ks_b), _ptr(planes), in_size, n, t, int(base).bit_length() - 1,
                   ctypes.addressof(registered))
        if not registered.value:
            return None
        # nb_ks_prepare replaced any earlier registration of ks_a: the finalizers of the earlier planes must leave
        # this one alone, so each registration carries its own token
        token = object()
        self._ks_registrations[ks_a.data_ptr()] = token
        for owner in (planes, ks_a, ks_b):
            weakref.finalize(owner, self._ks_forget, ks_a.data_ptr(), token)
        return planes

    def _ks_forget(self, ks_a_ptr, token):
        if self._ks_registrations.get(ks_a_ptr) is not token:
            return                                  # already dropped, or replaced by a later prepare of the key
        del self._ks_registrations[ks_a_ptr]
        if self.handle:
            self.lib.nb_ks_forget(self.handle, ctypes.c_void_p(ks_a_ptr))

    # --- the separate steps of the multi-kernel bootstrap (bootstrap.py:96-196) -------------------
    SHIFT_INVERT, SHIFT_MINUS_ONE, SHIFT_PLAIN = 0, 1, 2

    def shift_torus_polynomial(self, result, source, powers, power_idx=0, polys_per_power=1, mode=0):
        """result (polys, N) <- X^e * source; one power per `polys_per_power` polynomials, column `power_idx` of
        `powers` (rows of `powers.shape[-1]` entries when it is 2-D per group, else one entry per group)."""
        assert result.is_contiguous() and result.dtype == torch.int32
        source = self._dense(source, torch.int32)
        powers = self._dense(powers, torch.int32)
        n_poly = result.shape[-1]
        polys = result.numel() // n_poly
        groups = polys // polys_per_power
        stride = powers.numel() // groups
        self._call('nb_shift_torus_polynomial', _ptr(result), _ptr(source), _ptr(powers), stride, power_idx,
                   polys_per_power, mode, n_poly.bit_length() - 1, polys)
        return result

    def tlwe_noiseless_trivial(self, acc, cv, mu):
        assert acc.is_contiguous() and acc.dtype == torch.int32
        mu = self._dense(mu, torch.int32)
        n_poly, k1 = acc.shape[-1], acc.shape[-2]
        self._call('nb_tlwe_noiseless_trivial', _ptr(acc), _ptr(cv), _ptr(mu), k1 - 1, n_poly.bit_length() - 1,
                   acc.numel() // (k1 * n_poly))
        return acc

    def tlwe_extract_lwe_samples(self, out_a, out_b, acc):
        assert out_a.is_contiguous() and out_b.is_contiguous()
        acc = self._dense(acc, torch.int32)
        n_poly, k1 = acc.shape[-1], acc.shape[-2]
        self._call('nb_tlwe_extract_lwe_samples', _ptr(out_a), _ptr(out_b), _ptr(acc), k1 - 1,
                   n_poly.bit_length() - 1, acc.numel() // (k1 * n_poly))

    def tlwe_add_to(self, res, src, res_cv=None, src_cv=None):
        assert res.is_contiguous() and res.dtype == torch.int32
        src = self._dense(src, torch.int32)
        if res_cv is not None:
            assert res_cv.is_contiguous()
            src_cv = self._dense(src_cv, torch.float32)
        self._call('nb_tlwe_add_to', _ptr(res), _ptr(src), res.numel(), _ptr(res_cv), _ptr(src_cv),
                   0 if res_cv is None else res_cv.numel())

    def tgsw_decompose(self, acc, decomp_length, bs_log2_base, offset):
        """acc (..., N) int32 -> (..., l, N) digits (nb_tgsw_decompose)."""
        acc = self._dense(acc, torch.int32)
        n_poly = acc.shape[-1]
        out = self.empty(tuple(acc.shape[:-1]) + (decomp_length, n_poly), torch.int32)
        self._call('nb_tgsw_decompose', _ptr(out), _ptr(acc), acc.numel() // n_poly, decomp_length, bs_log2_base,
                   int(offset), n_poly.bit_length() - 1)
        return out

    def tgsw_mac(self, tr, bk_row, mask_size, decomp_length):
        """tr (B, k+1, l, 1024) u64, bk_row (k+1, l, k+1, 1024) u64 (reference layout) -> (B, k+1, 1024) u64."""
        tr = self._dense(tr, torch.int64)
        bk_row = self._dense(bk_row, torch.int64)
        batch = tr.numel() // ((mask_size + 1) * decomp_length * N)
        out = self.empty((batch, mask_size + 1, N), torch.int64)
        self._call('nb_tgsw_mac', _ptr(out), _ptr(tr), _ptr(bk_row), batch, mask_size, decomp_length)
        return out

    def t32_to_phase(self, out, messages, mspace_size):
        assert out.is_contiguous() and out.dtype == torch.int32
        messages = self._dense(messages, torch.int32)
        self._call('nb_t32_to_phase', _ptr(out), _ptr(messages), out.numel(), int(mspace_size))
        return out

    def lwe_dot(self, a, key, add1=None, add2=None, sign=1, out=None):
        """out[i] = add1[i] + add2[i] + sign * <a[i], key> in Torus32 (nb_lwe_dot); a (..., n), key (n,)."""
        a = self._dense(a, torch.int32)
        key = self._dense(key, torch.int32)
        n = key.numel()
        shape = tuple(a.shape[:-1])
        if out is None:
            out = self.empty(shape, torch.int32)
        assert out.is_contiguous() and out.dtype == torch.int32
        add1 = self._dense(add1, torch.int32) if add1 is not None else None
        add2 = self._dense(add2, torch.int32) if add2 is not None else None
        self._call('nb_lwe_dot', _ptr(out), _ptr(a), _ptr(key), _ptr(add1), _ptr(add2), int(sign), a.numel() // n, n)
        return out

    def make_keyswitch_key(self, ks_a, ks_b, ks_cv, in_key, out_key, noises_a, noises_b, log2_base, noise_variance):
        """Fill a key-switch key (nb_make_keyswitch_key); ks_a (in, t, base, n) etc. dense, updated in place."""
        assert ks_a.is_contiguous() and ks_b.is_contiguous() and ks_cv.is_contiguous()
        in_size, t, base, n = ks_a.shape
        self._call('nb_make_keyswitch_key', _ptr(ks_a), _ptr(ks_b), _ptr(ks_cv), _ptr(self._dense(in_key, torch.int32)),
                   _ptr(self._dense(out_key, torch.int32)), _ptr(self._dense(noises_a, torch.int32)),
                   _ptr(self._dense(noises_b, torch.int32)), in_size, n, t, int(log2_base),
                   ctypes.c_float(float(noise_variance)))

    def seeded_uniform(self, seed, nonce, shape, first=0):
        """Uniform Torus32 values of `shape` (int32): words [first, first + prod(shape)) of the ChaCha20 stream
        (seed, nonce) in C order (nb_seeded_uniform_i32).  `seed` holds 8 32-bit words (any integer dtype)."""
        seed = numpy.ascontiguousarray(numpy.asarray(seed).astype(numpy.int64).astype(numpy.uint32).reshape(-1))
        if seed.size != 8:
            raise ValueError('a seed is 8 32-bit words, got %d' % seed.size)
        out = self.empty(shape, torch.int32)
        if out.numel() == 0:
            return out
        self._call('nb_seeded_uniform_i32', seed.ctypes.data_as(ctypes.c_void_p), ctypes.c_uint64(int(nonce)),
                   ctypes.c_uint64(int(first)), _ptr(out), out.numel())
        return out

    def pk_prepare(self, a, b):
        """[A | b | 1] of a public key, a (m, n) and b (m,) int32, laid into the 4 byte planes that public_encrypt reads
        (nb_pk_prepare): a uint8 tensor of nb_pk_planes_bytes(m, n) bytes."""
        a = self._dense(a, torch.int32)
        b = self._dense(b, torch.int32)
        m, n = a.shape
        if b.shape != (m,):
            raise ValueError('public-key bodies of shape %s for %d rows' % (tuple(b.shape), m))
        planes = self.empty((self.lib.nb_pk_planes_bytes(m, n),), torch.uint8)
        self._call('nb_pk_prepare', _ptr(a), _ptr(b), m, n, _ptr(planes))
        return planes

    def public_encrypt(self, r_words, planes, m, n, mus, row_variance):
        """Public-key encryption of the B = mus.numel() messages `mus` (int32) with the random binary matrix R given as
        r_words (B, m/32) (bit i of row c = bit i % 32 of word (c, i // 32)) and `planes` from pk_prepare
        (nb_pk_encrypt).  Returns a (B, n), b (B,) int32 and the variances (B,) float32."""
        r_words = self._dense(r_words, torch.int32)
        mus = self._dense(mus, torch.int32).reshape(-1)
        planes = self._dense(planes, torch.uint8)
        batch = mus.numel()
        out_a, out_b = self.empty((batch, n), torch.int32), self.empty((batch,), torch.int32)
        out_cv = self.empty((batch,), torch.float32)
        if planes.numel() != self.lib.nb_pk_planes_bytes(m, n) or (m % 32 == 0 and r_words.numel() != batch * (m // 32)):
            raise ValueError('public_encrypt: %d plane bytes and %d R words do not fit m = %d, n = %d, %d messages'
                             % (planes.numel(), r_words.numel(), m, n, batch))
        if batch == 0:
            return out_a, out_b, out_cv
        self._call('nb_pk_encrypt', _ptr(r_words), _ptr(planes), m, n, _ptr(mus), ctypes.c_float(float(row_variance)),
                   _ptr(out_a), _ptr(out_b), _ptr(out_cv), batch)
        return out_a, out_b, out_cv

    def pack_digits(self, a):
        """LWE masks a (B, n) int32 -> digit polynomials (ceil(B / N), 2 n, N) int32: row 2 i + j of group g holds digit
        j of a[g N + p][i] at coefficient p, 0 in the empty slots (nb_pack_digits)."""
        a = self._dense(a, torch.int32)
        batch, n = a.shape
        out = self.empty(((batch + N - 1) // N, 2 * n, N), torch.int32)
        if batch:
            self._call('nb_pack_digits', _ptr(a), n, _ptr(out), batch)
        return out

    def ntt_mac(self, x, key):
        """out (G, U, N) = sum_r x (G, R, N) . key (R, U, N) on plain-form field elements (nb_ntt_mac)."""
        x = self._dense(x, torch.int64)
        key = self._dense(key, torch.int64)
        if x.dim() != 3 or key.dim() != 3 or x.shape[2] != N or key.shape[2] != N or x.shape[1] != key.shape[0]:
            raise ValueError('ntt_mac: x %s and key %s are not (G, R, N) and (R, U, N)' % (tuple(x.shape), tuple(key.shape)))
        groups, rows = x.shape[:2]
        outs = key.shape[1]
        out = self.empty((groups, outs, N), torch.int64)
        if groups:
            self._call('nb_ntt_mac', _ptr(x), _ptr(key), _ptr(out), rows, outs, groups)
        return out

    def pack_finish(self, c, b):
        """c (G, k+1, N) int32 and the bodies b (B,) int32 -> (G, k+1, N) uint16: round_16(-c) for the masks,
        round_16(b[g N + p] - c) at the slots of the body (nb_pack_finish)."""
        c = self._dense(c, torch.int32)
        b = self._dense(b, torch.int32).reshape(-1)
        groups, k1 = c.shape[0], c.shape[1]
        batch = b.numel()
        if c.dim() != 3 or c.shape[2] != N or groups != (batch + N - 1) // N:
            raise ValueError('pack_finish: %s polynomials for %d bodies' % (tuple(c.shape), batch))
        out = self.empty(tuple(c.shape), torch.uint16)
        if batch:
            self._call('nb_pack_finish', _ptr(c), _ptr(b), k1 - 1, _ptr(out), batch)
        return out

    def compact_finish(self, c, e1, e2, mus):
        """The products c (G, k+1, N) int32, the noises e1 (G, k, N) and e2 (G, N) and the messages mus (B,) int32 ->
        compact data (G, k+1, N) uint16: round_16(c + e1) for the masks, round_16(c + e2 + mu) at the occupied slots of
        the body, 0 at its empty slots (nb_compact_finish)."""
        c = self._dense(c, torch.int32)
        e1 = self._dense(e1, torch.int32)
        e2 = self._dense(e2, torch.int32)
        mus = self._dense(mus, torch.int32).reshape(-1)
        batch = mus.numel()
        if c.dim() != 3 or c.shape[2] != N or c.shape[0] != (batch + N - 1) // N:
            raise ValueError('compact_finish: %s products for %d messages' % (tuple(c.shape), batch))
        groups, k1 = c.shape[0], c.shape[1]
        if tuple(e1.shape) != (groups, k1 - 1, N) or tuple(e2.shape) != (groups, N):
            raise ValueError('compact_finish: noises %s and %s for products %s'
                             % (tuple(e1.shape), tuple(e2.shape), tuple(c.shape)))
        out = self.empty(tuple(c.shape), torch.uint16)
        if batch:
            self._call('nb_compact_finish', _ptr(c), _ptr(e1), _ptr(e2), _ptr(mus), k1 - 1, _ptr(out), batch)
        return out

    def compact_extract(self, data, rows):
        """Compact data (G, k+1, N) uint16 -> the LWE samples of its first `rows` slots under the extracted key of S:
        a (rows, k N) and b (rows,) int32, every coefficient shifted back by 16 bits (nb_compact_extract)."""
        data = self._dense(data, torch.uint16)
        if data.dim() != 3 or data.shape[2] != N or data.shape[0] != (rows + N - 1) // N:
            raise ValueError('compact_extract: data %s for %d rows' % (tuple(data.shape), rows))
        k1 = data.shape[1]
        out_a, out_b = self.empty((rows, (k1 - 1) * N), torch.int32), self.empty((rows,), torch.int32)
        if rows:
            self._call('nb_compact_extract', _ptr(data), k1 - 1, _ptr(out_a), _ptr(out_b), rows)
        return out_a, out_b

    def tree_prepare(self, masks, body):
        """The tree key's masks (n, t, k, N) and bodies (n, t, N) int32 laid into the 4 byte planes that tree_keyswitch
        reads (nb_tree_prepare): a uint8 tensor of nb_tree_planes_bytes(n, k) bytes."""
        masks = self._dense(masks, torch.int32)
        body = self._dense(body, torch.int32)
        n, t, k, n_poly = masks.shape
        if t != 2 or n_poly != N or tuple(body.shape) != (n, t, N):
            raise ValueError('tree_prepare: masks %s and bodies %s are not (n, 2, k, N) and (n, 2, N)'
                             % (tuple(masks.shape), tuple(body.shape)))
        planes = self.empty((self.lib.nb_tree_planes_bytes(n, k),), torch.uint8)
        self._call('nb_tree_prepare', _ptr(masks), _ptr(body), n, k, _ptr(planes))
        return planes

    def tree_keyswitch(self, a, planes, mask_size):
        """LWE masks a (R, n) int32 -> V (R, k+1, N) int32, V = sum_ij d_ij(a) T_ij mod 2^32 (nb_tree_keyswitch)."""
        a = self._dense(a, torch.int32)
        planes = self._dense(planes, torch.uint8)
        rows, n = a.shape
        if planes.numel() != self.lib.nb_tree_planes_bytes(n, int(mask_size)):
            raise ValueError('tree_keyswitch: %d plane bytes do not fit n = %d, k = %d' % (planes.numel(), n, mask_size))
        out = self.empty((rows, mask_size + 1, N), torch.int32)
        if rows:
            self._call('nb_tree_keyswitch', _ptr(a), _ptr(planes), n, int(mask_size), _ptr(out), rows)
        return out

    def tree_assemble(self, v, b, bits):
        """v (T, 2^bits, k+1, N) and bodies b (T, 2^bits) int32 -> test vectors (T, k+1, N) (nb_tree_assemble)."""
        v = self._dense(v, torch.int32)
        b = self._dense(b, torch.int32)
        if v.dim() != 4 or v.shape[1] != 1 << int(bits) or v.shape[3] != N or tuple(b.shape) != tuple(v.shape[:2]):
            raise ValueError('tree_assemble: v %s and b %s do not fit %d-bit digits'
                             % (tuple(v.shape), tuple(b.shape), bits))
        count, _, k1, _ = v.shape
        out = self.empty((count, k1, N), torch.int32)
        if count:
            self._call('nb_tree_assemble', _ptr(v), _ptr(b), int(bits), k1 - 1, _ptr(out), count)
        return out

    def bootstrap_glwe_lut_extract(self, x, tv, bk_int):
        """The programmable bootstrap of x = (a (B, n), b (B,)) with per-ciphertext GLWE test vectors tv (B, 2, N):
        returns the extracted samples a (B, N), b (B,) (nb_bootstrap_glwe_lut_extract)."""
        a, b = self._dense(x[0], torch.int32), self._dense(x[1], torch.int32)
        tv = self._dense(tv, torch.int32)
        B = b.numel()
        n = a.shape[-1]
        if tuple(tv.shape) != (B, 2, N) or a.numel() != B * n:
            raise ValueError('bootstrap_glwe_lut_extract: tv %s for %d ciphertexts' % (tuple(tv.shape), B))
        out_a, out_b = self.empty((B, N), torch.int32), self.empty((B,), torch.int32)
        self._call('nb_bootstrap_glwe_lut_extract', _ptr(a), _ptr(b), _ptr(tv), _ptr(bk_int), n, _ptr(out_a),
                   _ptr(out_b), B)
        return out_a, out_b

    # --- encrypted-index lookups (nufhe_b200/index_lookup.py) -----------------------------------
    def index_prepare(self, ggsw):
        """Selector rows (..., 2, 2, 2, N) int32 -> their FP64 spectra (rows, nb_bk_multibit_row_u64()) (nb_index_prepare)."""
        ggsw = self._dense(ggsw, torch.int32)
        rows = ggsw.numel() // (8 * N)
        out = self.empty((rows, self.lib.nb_bk_multibit_row_u64()), torch.int64)
        if rows:
            self._call('nb_index_prepare', _ptr(ggsw), rows, _ptr(out))
        return out

    @staticmethod
    def _index_nodes(x, queries, what):
        """(nodes, stride): x (queries, nodes, 2, N) per query, or (nodes, 2, N) shared by all queries (stride 0)."""
        if x.shape[-2:] != (2, N) or x.dim() not in (3, 4) or (x.dim() == 4 and x.shape[0] != queries):
            raise ValueError('%s: %s GLWE samples for %d queries' % (what, tuple(x.shape), queries))
        return x.shape[-3], (0 if x.dim() == 3 else x.shape[1] * 2 * N)

    @staticmethod
    def _index_sel(sel, bit, queries, what):
        if sel.dim() != 3 or sel.shape[0] != queries or not 0 <= bit < sel.shape[1]:
            raise ValueError('%s: selector spectra %s for %d queries, bit %d' % (what, tuple(sel.shape), queries, bit))
        return ctypes.c_void_p(sel.data_ptr() + bit * sel.shape[2] * sel.element_size()), sel.shape[1] * sel.shape[2]

    def index_cmux_level(self, x, sel, bit, queries):
        """One CMux-tree level (nb_index_cmux_level): out[q][i] = x[q][2i] + C [x] (x[q][2i+1] - x[q][2i]) with C the
        selector `bit` of query q in sel (queries, m, R) (index_prepare); x (queries, 2 nodes, 2, N) or (2 nodes, 2, N)
        shared by every query.  Returns (queries, nodes, 2, N)."""
        x = self._dense(x, torch.int32)
        sel = self._dense(sel, torch.int64)
        pairs, stride = self._index_nodes(x, queries, 'index_cmux_level')
        if pairs % 2:
            raise ValueError('index_cmux_level: an odd node count %d' % pairs)
        sp, sstride = self._index_sel(sel, bit, queries, 'index_cmux_level')
        out = self.empty((queries, pairs // 2, 2, N), torch.int32)
        if queries and pairs:
            self._call('nb_index_cmux_level', _ptr(x), stride, sp, sstride, _ptr(out), pairs // 2, queries)
        return out

    def index_rotate_extract(self, acc, sel, bits, columns, queries):
        """Rotation by the low index bits and extraction (nb_index_rotate_extract): acc (queries, A, 2, N) or (A, 2, N)
        shared, A = columns for bits >= 10, else 1; sel (queries, bits, R).  Returns a (columns, queries, N) and
        b (columns, queries)."""
        acc = self._dense(acc, torch.int32)
        sel = self._dense(sel, torch.int64)
        accs, stride = self._index_nodes(acc, queries, 'index_rotate_extract')
        if accs != (columns if bits >= 10 else 1) or sel.dim() != 3 or sel.shape[1] != bits:
            raise ValueError('index_rotate_extract: %d accumulators and %s selector spectra for %d columns of %d bits'
                             % (accs, tuple(sel.shape), columns, bits))
        sp, sstride = self._index_sel(sel, 0, queries, 'index_rotate_extract')
        out_a, out_b = self.empty((columns, queries, N), torch.int32), self.empty((columns, queries), torch.int32)
        if queries:
            self._call('nb_index_rotate_extract', _ptr(acc), stride, sp, sstride, int(bits), columns, _ptr(out_a),
                       _ptr(out_b), queries)
        return out_a, out_b

    @staticmethod
    def _index_tables(tables, table_ids, queries, what):
        """(tables per call, nodes per table, stride, ids): tables (T, nodes, 2, N), table_ids (queries,) < T."""
        ids = numpy.ascontiguousarray(table_ids, numpy.uint32).reshape(-1)
        if tables.dim() != 4 or tables.shape[-2:] != (2, N) or ids.size != queries:
            raise ValueError('%s: tables %s and %d table ids for %d queries' % (what, tuple(tables.shape), ids.size, queries))
        return tables.shape[0], tables.shape[1], tables.shape[1] * 2 * N, ids

    def index_cmux_level_indirect(self, tables, table_ids, sel, bit, queries):
        """index_cmux_level with query q reading tables[table_ids[q]] (nb_index_cmux_level_indirect): tables
        (T, 2 nodes, 2, N), table_ids a host array of `queries` ids.  Returns (queries, nodes, 2, N)."""
        tables = self._dense(tables, torch.int32)
        sel = self._dense(sel, torch.int64)
        count, pairs, stride, ids = self._index_tables(tables, table_ids, queries, 'index_cmux_level_indirect')
        if pairs % 2:
            raise ValueError('index_cmux_level_indirect: an odd node count %d' % pairs)
        sp, sstride = self._index_sel(sel, bit, queries, 'index_cmux_level_indirect')
        out = self.empty((queries, pairs // 2, 2, N), torch.int32)
        if queries and pairs:
            self._call('nb_index_cmux_level_indirect', _ptr(tables), stride, count, ids.ctypes.data_as(ctypes.c_void_p),
                       sp, sstride, _ptr(out), pairs // 2, queries)
        return out

    def index_rotate_extract_indirect(self, tables, table_ids, sel, bits, columns, queries):
        """index_rotate_extract with query q reading tables[table_ids[q]] (nb_index_rotate_extract_indirect): tables
        (T, A, 2, N), A = columns for bits >= 10, else 1.  Returns a (columns, queries, N) and b (columns, queries)."""
        tables = self._dense(tables, torch.int32)
        sel = self._dense(sel, torch.int64)
        count, accs, stride, ids = self._index_tables(tables, table_ids, queries, 'index_rotate_extract_indirect')
        if accs != (columns if bits >= 10 else 1) or sel.dim() != 3 or sel.shape[1] != bits:
            raise ValueError('index_rotate_extract_indirect: %d accumulators and %s selector spectra for %d columns of %d '
                             'bits' % (accs, tuple(sel.shape), columns, bits))
        sp, sstride = self._index_sel(sel, 0, queries, 'index_rotate_extract_indirect')
        out_a, out_b = self.empty((columns, queries, N), torch.int32), self.empty((columns, queries), torch.int32)
        if queries:
            self._call('nb_index_rotate_extract_indirect', _ptr(tables), stride, count,
                       ids.ctypes.data_as(ctypes.c_void_p), sp, sstride, int(bits), columns, _ptr(out_a), _ptr(out_b),
                       queries)
        return out_a, out_b

    # --- oblivious writes (nufhe_b200/index_write.py) ---------------------------------------------
    def index_write_assemble(self, v, b, bits):
        """The delta of every query (nb_index_write_assemble): v (Q, W, 2, N) tree_keyswitch output or None for trivial
        values, bodies b (Q, W) int32.  Returns (Q, A, 2, N), A = W for bits >= 10, else 1."""
        b = self._dense(b, torch.int32)
        if b.dim() != 2:
            raise ValueError('index_write_assemble: bodies %s are not (queries, columns)' % (tuple(b.shape),))
        Q, W = b.shape
        if v is not None:
            v = self._dense(v, torch.int32)
            if tuple(v.shape) != (Q, W, 2, N):
                raise ValueError('index_write_assemble: v %s for bodies %s' % (tuple(v.shape), tuple(b.shape)))
        out = self.empty((Q, W if bits >= 10 else 1, 2, N), torch.int32)
        if Q:
            self._call('nb_index_write_assemble', _ptr(v), _ptr(b), int(bits), W, _ptr(out), Q)
        return out

    @staticmethod
    def _write_tables(acc, table_ids, queries, what):
        """(acc, stride, count, ids) of the accumulators acc (T, P, 2, N) int32 and the host ids (queries,) < T (None:
        one table)."""
        if acc is None:
            return None, 0, 0, None
        if acc.dim() != 4 or acc.shape[-2:] != (2, N) or not acc.is_contiguous() or acc.dtype != torch.int32:
            raise ValueError('%s: accumulators %s %s are not contiguous int32 (T, P, 2, N)' % (what, acc.dtype, tuple(acc.shape)))
        ids = None
        if table_ids is not None:
            ids = numpy.ascontiguousarray(table_ids, numpy.uint32).reshape(-1)
            if ids.size != queries:
                raise ValueError('%s: %d table ids for %d queries' % (what, ids.size, queries))
        return acc, acc.shape[1] * 2 * N, acc.shape[0], ids

    def index_write_rotate(self, delta, sel, bits, acc=None, table_ids=None):
        """The rotation by X^(+idx mod 1024) of every delta (nb_index_write_rotate): delta (Q, A, 2, N), sel (Q, bits, R).
        bits > 10: returns the rotated (Q, A, 2, N); bits <= 10: adds them into the accumulators acc (T, P, 2, N) in
        place, query q into acc[table_ids[q]] (None: T = 1), and returns None."""
        delta = self._dense(delta, torch.int32)
        sel = self._dense(sel, torch.int64)
        Q, A = delta.shape[0], delta.shape[1]
        if delta.dim() != 4 or delta.shape[-2:] != (2, N) or sel.dim() != 3 or sel.shape[1] != bits:
            raise ValueError('index_write_rotate: deltas %s and selector spectra %s for %d bits'
                             % (tuple(delta.shape), tuple(sel.shape), bits))
        columns = A if bits >= 10 else 1
        sp, sstride = self._index_sel(sel, 0, Q, 'index_write_rotate')
        acc, astride, count, ids = self._write_tables(acc, table_ids, Q, 'index_write_rotate')
        out = self.empty((Q, A, 2, N), torch.int32) if acc is None else None
        if Q:
            self._call('nb_index_write_rotate', _ptr(delta), sp, sstride, int(bits), columns, _ptr(out), _ptr(acc),
                       astride, count, None if ids is None else ids.ctypes.data_as(ctypes.c_void_p), Q)
        return out

    def index_demux_level(self, x, sel, bit, acc=None, table_ids=None):
        """One demultiplexer level (nb_index_demux_level): node y of x (Q, K, 2, N) becomes (y - C [x] y, C [x] y), C
        the selector `bit` of sel (Q, m, R).  Returns (Q, 2 K, 2, N), or with acc (the last level) adds them into
        acc[table_ids[q]] in place and returns None."""
        x = self._dense(x, torch.int32)
        sel = self._dense(sel, torch.int64)
        if x.dim() != 4 or x.shape[-2:] != (2, N):
            raise ValueError('index_demux_level: %s GLWE samples' % (tuple(x.shape),))
        Q, K = x.shape[0], x.shape[1]
        sp, sstride = self._index_sel(sel, bit, Q, 'index_demux_level')
        acc, astride, count, ids = self._write_tables(acc, table_ids, Q, 'index_demux_level')
        out = self.empty((Q, 2 * K, 2, N), torch.int32) if acc is None else None
        if Q and K:
            self._call('nb_index_demux_level', _ptr(x), sp, sstride, _ptr(out), _ptr(acc), astride, count,
                       None if ids is None else ids.ctypes.data_as(ctypes.c_void_p), K, Q)
        return out

    def lwe_affine(self, res, x1, x2, c, s1, s2):
        res_a, res_b = res
        B = res_b.numel()
        n = res_a.shape[-1]
        a1 = b1 = a2 = b2 = None
        if x1 is not None:
            a1, b1 = self._dense(x1[0], torch.int32), self._dense(x1[1], torch.int32)
        if x2 is not None:
            a2, b2 = self._dense(x2[0], torch.int32), self._dense(x2[1], torch.int32)
        self._call('nb_lwe_affine', _ptr(res_a), _ptr(res_b), _ptr(a1), _ptr(b1), _ptr(a2), _ptr(b2),
                   int(c), int(s1), int(s2), B, n)
        return res


class DeviceParams:
    """The few fields of Reikna's device_params that PerformanceParameters.for_device() looks at
    (nufhe/performance.py:137-236)."""

    def __init__(self, device):
        props = torch.cuda.get_device_properties(device)
        self.compute_units = props.multi_processor_count
        self.max_work_group_size = 1024
        self.local_mem_size = 227 * 1024
        self.name = props.name
