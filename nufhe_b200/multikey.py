"""Gates and lookup tables on ciphertexts of many cloud keys in one fused launch (DESIGN.md section 17).

A server with many clients holds one cloud key per client ("tenant") and, at any moment, a few ciphertexts per key.
A VirtualMachine per key would bootstrap each handful in a launch of its own, leaving most of the GPU idle; a
MultiKeyVirtualMachine concatenates the operands of every tenant and runs one multi-key bootstrap (each ciphertext with
its own tenant's bootstrapping key) and one multi-key key switch.  Every output is bit-identical to what that tenant's
own VirtualMachine returns for the same operands.
"""
import numpy
import torch

from .api_low_level import NuFHECloudKey, empty_ciphertext
from .gates import MU, _BINARY_GATES, check_shape, get_shape, result_shape
from .lwe import LweSampleArray
from .lut import _check_config, _check_margin, _sigma
from .numeric_functions import phase_to_t32
from .performance import PerformanceParameters
from .tgsw import engine_format, fused_kernel_supported
from . import gates

# gates that need no key: run per tenant
_KEYLESS = {'not': 1, 'copy': 1, 'constant': 1}


class MultiKeyVirtualMachine:
    """Executes gates and one-table LUTs on the ciphertexts of several cloud keys at once.

    Every operand is a list aligned with `cloud_keys`: entry t holds tenant t's ciphertexts (of any shape, broadcast per
    tenant as VirtualMachine does), or None when tenant t has no work, in which case all its operands must be None.
    The result is a list aligned the same way (None for idle tenants).

    .. method:: gate_<operator>(*operand_lists, dest=None)
    """

    def __init__(self, thread, cloud_keys, perf_params: PerformanceParameters = None):
        cloud_keys = list(cloud_keys)
        if not cloud_keys:
            raise ValueError('a multi-key machine needs at least one cloud key')
        for t, key in enumerate(cloud_keys):
            if not isinstance(key, NuFHECloudKey):
                raise TypeError('tenant %d: a multi-key machine takes NuFHECloudKey objects (decompress a compressed key '
                                'first), got %s' % (t, type(key).__name__))
        params = cloud_keys[0].params
        pp = (perf_params if perf_params is not None else PerformanceParameters(params)).for_device(thread.device_params)
        for t, key in enumerate(cloud_keys):
            if key.params != params:
                raise ValueError('tenant %d: the cloud key was made for other parameters than tenant 0\'s' % t)
            bk = key.bootstrap_key
            if getattr(bk, 'multi_bit', 1) == 2:
                raise ValueError('tenant %d: multi-bit bootstrap keys are not supported by the multi-key machine' % t)
            if not pp.single_kernel_bootstrap or not fused_kernel_supported(bk.bk_params):
                raise ValueError('tenant %d: the multi-key machine runs the fused bootstrap only (single_kernel_bootstrap=True, '
                                 'tlwe_mask_size=1)' % t)
        self.thread = thread
        self.params = params
        self.cloud_keys = cloud_keys
        self.perf_params = pp
        # lay the keys out for the fused kernel and the tensor-core key switch once, as VirtualMachine does
        self._bk_ints = [engine_format(thread, key.bootstrap_key.tgsw) for key in cloud_keys]
        for key in cloud_keys:
            key.keyswitch_key.prepare_gemm(thread)
        self._ks = [key.keyswitch_key.device_arrays() for key in cloud_keys]
        # an empty launch checks every key on the engine (FP64 spectra, not a multi-bit range)
        n = params.in_out_params.size
        empty = (thread.empty((0, n), torch.int32), thread.empty((0,), torch.int32))
        try:
            thread.mk_bootstrap_extract(empty, None, 0, 1, 0, MU, self._bk_ints, [0] * len(cloud_keys))
        except ValueError as e:
            raise ValueError('a cloud key cannot run in a multi-key launch: %s' % e) from None

    @property
    def tenants(self):
        return len(self.cloud_keys)

    def empty_ciphertext(self, shape):
        return empty_ciphertext(self.thread, self.params, shape)

    # --- operands ------------------------------------------------------------------------------
    def _active(self, operand_lists, dest):
        """Validate the operand lists; returns the tenants with work and, for each, its result shape."""
        T = self.tenants
        for i, ops in enumerate(operand_lists):
            if not isinstance(ops, (list, tuple)) or len(ops) != T:
                raise ValueError('operand %d must be a list of %d entries, one per tenant' % (i, T))
        if dest is not None and (not isinstance(dest, (list, tuple)) or len(dest) != T):
            raise ValueError('dest must be a list of %d entries, one per tenant' % T)
        active, shapes = [], {}
        for t in range(T):
            present = [ops[t] is not None for ops in operand_lists]
            if not any(present):
                if dest is not None and dest[t] is not None:
                    raise ValueError('tenant %d has no operands but a destination' % t)
                continue
            if not all(present):
                raise ValueError('tenant %d: operands must all be given or all be None' % t)
            shape = result_shape(*[get_shape(ops[t]) for ops in operand_lists])
            if dest is not None:
                if dest[t] is None:
                    raise ValueError('tenant %d has operands but no destination' % t)
                check_shape(dest[t], *[ops[t] for ops in operand_lists])
                shape = tuple(dest[t].shape)
            active.append(t)
            shapes[t] = shape
        return active, shapes

    @staticmethod
    def _expand(x, shape):
        a, b = x.a, x.b
        if tuple(b.shape) != shape:
            while b.dim() < len(shape):
                a, b = a.unsqueeze(0), b.unsqueeze(0)
            a, b = a.expand(shape + (a.shape[-1],)), b.expand(shape)
        return a.contiguous().reshape(-1, a.shape[-1]), b.contiguous().reshape(-1)

    def _concat(self, ops, active, shapes):
        parts = [self._expand(ops[t], shapes[t]) for t in active]
        return torch.cat([p[0] for p in parts]), torch.cat([p[1] for p in parts])

    def _counts(self, active, shapes):
        counts = [0] * self.tenants
        for t in active:
            counts[t] = int(numpy.prod(shapes[t], dtype=numpy.int64))
        return counts

    def _keyswitch(self, counts, src1, src2=None, c=0):
        return self.thread.mk_keyswitch(self._ks, counts, src1, src2, c=c, want_cv=True)

    def _results(self, res, active, shapes, counts, dest):
        """Tenant views of one key-switch result (res_a, res_b, res_cv), or copies into `dest`."""
        ra, rb, rcv = res
        out = [None] * self.tenants
        row = 0
        for t in active:
            B, shape = counts[t], shapes[t]
            a = ra[row:row + B].reshape(shape + (ra.shape[-1],))
            b, cv = rb[row:row + B].reshape(shape), rcv[row:row + B].reshape(shape)
            row += B
            if dest is None:
                out[t] = LweSampleArray(self.params.in_out_params, a, b, cv)
            else:
                dest[t].a.copy_(a)
                dest[t].b.copy_(b)
                dest[t].current_variances.copy_(cv)
                out[t] = dest[t]
        return out

    # --- gates ---------------------------------------------------------------------------------
    def _binary(self, name, a, b, dest):
        active, shapes = self._active((a, b), dest)
        if not active:
            return [None] * self.tenants
        num, den, sa, sb = _BINARY_GATES[name]
        counts = self._counts(active, shapes)
        ext = self.thread.mk_bootstrap_extract(self._concat(a, active, shapes), self._concat(b, active, shapes),
                                               phase_to_t32(num, den), sa, sb, MU, self._bk_ints, counts)
        return self._results(self._keyswitch(counts, ext), active, shapes, counts, dest)

    def _mux(self, a, b, c, dest):
        active, shapes = self._active((a, b, c), dest)
        if not active:
            return [None] * self.tenants
        counts = self._counts(active, shapes)
        pa, pb, pc = (self._concat(x, active, shapes) for x in (a, b, c))
        and_const = phase_to_t32(-1, 8)
        # AND(a, b) and AND(not a, c) as two jobs of one launch, then one key switch of (0,1/8) + u1 + u2 (gates.gate_mux)
        u1, u2 = self.thread.mk_bootstrap_extract2((pa, pb, and_const, 1, 1), (pa, pc, and_const, -1, 1), MU,
                                                   self._bk_ints, counts)
        return self._results(self._keyswitch(counts, u1, u2, c=phase_to_t32(1, 8)), active, shapes, counts, dest)

    def _keyless(self, name, args, dest):
        active, shapes = self._active(args, dest)
        out = [None] * self.tenants
        for t in active:
            r = dest[t] if dest is not None else self.empty_ciphertext(shapes[t])
            getattr(gates, 'gate_' + name)(self.thread, self.cloud_keys[t], r, *[ops[t] for ops in args],
                                           perf_params=self.perf_params)
            out[t] = r
        return out

    def _gate(self, name, *args, dest=None):
        if name in _BINARY_GATES:
            arity = 2
        elif name == 'mux':
            arity = 3
        elif name in _KEYLESS:
            arity = _KEYLESS[name]
        else:
            raise AttributeError('gate_' + name)
        if len(args) != arity:
            raise TypeError('gate_%s takes %d operand lists, got %d' % (name, arity, len(args)))
        if name in _KEYLESS:
            if name == 'constant':
                # values, not ciphertexts: shapes come from the values themselves
                args = ([None if v is None else numpy.asarray(v) for v in args[0]],)
            return self._keyless(name, args, dest)
        if name == 'mux':
            return self._mux(*args, dest)
        return self._binary(name, *args, dest)

    def __getattr__(self, name):
        if name.startswith('gate_'):
            gate = name[len('gate_'):]
            if gate in _BINARY_GATES or gate == 'mux' or gate in _KEYLESS:
                return lambda *args, **kwds: self._gate(gate, *args, **kwds)
        raise AttributeError(name)

    # --- lookup tables -------------------------------------------------------------------------
    def lut(self, table, xs, ys=None, shift=0, dest=None):
        """f(x), or f(x * 2^shift + y), for every tenant's ciphertexts with one LookupTable (VirtualMachine.make_lut)
        shared by all tenants.  Entry t of the result is one ciphertext array, or a list of 2^L of them for a table with
        several outputs.  ValueError for a configuration without enough noise margin (lut.check_noise) and for tables
        with one entry per ciphertext."""
        if table.batch_shape:
            raise ValueError('the multi-key machine takes one table for every ciphertext, not one per ciphertext')
        operand_lists = (xs,) if ys is None else (xs, ys)
        K = table.outputs
        L = table.log2_outputs
        dest_lists = None
        if dest is not None:
            if not isinstance(dest, (list, tuple)) or len(dest) != self.tenants:
                raise ValueError('dest must be a list of %d entries, one per tenant' % self.tenants)
            dest_lists = [None if d is None else ([d] if isinstance(d, LweSampleArray) else list(d)) for d in dest]
            for t, d in enumerate(dest_lists):
                if d is not None and len(d) != K:
                    raise ValueError('tenant %d: a table with %d outputs needs %d results, got %d' % (t, K, K, len(d)))
        active, shapes = self._active(operand_lists, None if dest_lists is None else
                                      [None if d is None else d[0] for d in dest_lists])
        # the noise rule of VirtualMachine.lut (every tenant has the same parameters)
        bk, ks = self.cloud_keys[0].bootstrap_key, self.cloud_keys[0].keyswitch_key
        sh = None if ys is None else shift
        _check_config(table.bits, L, sh)
        _check_margin(_sigma(bk.in_out_params, bk.bk_params, ks.decomp_length, ks.log2_base, L, sh), table.bits, L, sh)
        out = [None] * self.tenants
        if not active:
            return out
        counts = self._counts(active, shapes)
        p1 = self._concat(xs, active, shapes)
        p2 = self._concat(ys, active, shapes) if ys is not None else None
        s1 = 1 << shift if ys is not None else 1
        ea, eb = self.thread.mk_bootstrap_lut_extract(p1, p2, 0, s1, 1, table.tv, L, self._bk_ints, counts)
        ra, rb, rcv = self._keyswitch([c * K for c in counts], (ea, eb))
        # sample j of ciphertext c is row c * K + j: one contiguous block per output
        total = rb.numel() // K
        ra = ra.reshape(total, K, -1).transpose(0, 1).contiguous()
        rb = rb.reshape(total, K).t().contiguous()
        rcv = rcv.reshape(total, K).t().contiguous()
        per_output = [self._results((ra[j], rb[j], rcv[j]), active, shapes, counts,
                                    None if dest_lists is None else [None if d is None else d[j] for d in dest_lists])
                      for j in range(K)]
        for t in active:
            out[t] = per_output[0][t] if K == 1 else [per_output[j][t] for j in range(K)]
        return out
