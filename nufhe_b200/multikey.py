"""Gates and lookup tables on ciphertexts of many cloud keys in one fused launch (DESIGN.md section 17).

A server with many clients holds one cloud key per client ("tenant") and, at any moment, a few ciphertexts per key.
A VirtualMachine per key would bootstrap each handful in a launch of its own, leaving most of the GPU idle; a
MultiKeyVirtualMachine concatenates the operands of every tenant and runs one multi-key bootstrap (each ciphertext with
its own tenant's bootstrapping key) and one multi-key key switch.  Every output is bit-identical to what that tenant's
own VirtualMachine returns for the same operands.

With `resident_tenants=R` the machine takes compressed cloud keys instead and keeps at most R of them expanded on the
device (DESIGN.md section 19): an operation runs in rounds of at most R tenants, each round first expanding the keys it
lacks into slots freed by the least recently used tenants.
"""
import collections
import functools
import inspect

import numpy
import torch

from .api_low_level import NuFHECloudKey, empty_ciphertext
from .compressed import CompressedCloudKey
from .gates import MU, _BINARY_GATES, check_shape, get_shape, result_shape
from .lwe import LweSampleArray
from .lut import LookupTable, _check_config, _check_margin, _expand, _sigma
from .numeric_functions import phase_to_t32
from .performance import PerformanceParameters
from .tgsw import engine_format, fused_kernel_supported
from .tree_lut import NuFHETreeKey, TreeLookupTable
from .packing import NuFHEPackingKey, PackedLweSampleArray
from .compact import CompactLweSampleArray
from .index_lookup import EncryptedIndexArray, EncryptedIndexTable, IndexTable
from .batch_keys import TenantKeys
from . import compact, gates, index_lookup, index_write, packing, tree_lut

# gates that need no key: run per tenant
_KEYLESS = {'not': 1, 'copy': 1, 'constant': 1}


def _in_rounds(operands, masked=()):
    """Run a method of a machine on compressed keys in rounds (DESIGN.md section 19).  `operands` name the arguments
    that hold one entry per tenant whose non-None entries make a tenant active (`digits`: a list of such lists);
    `masked` name further per-tenant arguments.  Each round calls the method with every per-tenant argument masked to
    the round's tenants and the round's keys in place; tenants are independent, so the rounds do not change a result.
    A call whose per-tenant arguments are malformed goes straight to the method, which raises."""
    def wrap(method):
        sig = inspect.signature(method)

        @functools.wraps(method)
        def run(self, *args, **kwds):
            if self._pool is None:
                return method(self, *args, **kwds)
            call = sig.bind(self, *args, **kwds)
            T = self.tenants

            def lists(name):
                x = call.arguments.get(name)
                if x is None or (name == 'table' and not isinstance(x, (list, tuple))):
                    return []
                return list(x) if name == 'digits' else [x]
            per_tenant = [x for name in operands + masked for x in lists(name)]
            if any(not isinstance(x, (list, tuple)) or len(x) != T for x in per_tenant):
                return method(self, *args, **kwds)
            active = [t for t in range(T) if any(x[t] is not None for name in operands for x in lists(name))]
            out = [None] * T
            for keep in self._pool.rounds(active):
                self._pool.fill(self, keep)
                keep = set(keep)
                masked_call = sig.bind(self, *args, **kwds)
                for name in operands + masked:
                    x = masked_call.arguments.get(name)
                    if not lists(name):
                        continue
                    mask = lambda lst: [v if t in keep else None for t, v in enumerate(lst)]
                    masked_call.arguments[name] = [mask(d) for d in x] if name == 'digits' else mask(x)
                res = method(*masked_call.args, **masked_call.kwargs)
                for t in keep:
                    out[t] = res[t]
            return out
        return run
    return wrap


class _SlotPool:
    """The expanded keys of a machine on compressed cloud keys: at most R slots, each the engine-row bootstrap key
    (FP64 part only) and the key-switch masks of one tenant, allocated lazily and reused in least-recently-used order.
    While a round runs, the machine's per-tenant key lists point at the round's slots.  The pool holds no reference to
    its machine, so the slots go with the machine."""

    def __init__(self, keys, R):
        self.keys = keys
        self.R = R
        self.lru = collections.OrderedDict()           # tenant -> (bk slot, ks_a), least recently used first
        self.slots = 0
        # ks_cv of decompress(): 0 for rows h = 0, the key's variance elsewhere; one per distinct variance
        self.ks_cv = {}
        for key in keys:
            if key.ks_variance not in self.ks_cv:
                cv = torch.zeros(tuple(key.ks_b.shape), dtype=torch.float32, device=key.ks_b.device)
                cv[:, :, 1:] = key.ks_variance
                self.ks_cv[key.ks_variance] = cv

    def rounds(self, active):
        """The active tenants that hold a slot, in tenant order, then the others, R at a time."""
        order = [t for t in active if t in self.lru] + [t for t in active if t not in self.lru]
        return [order[i:i + self.R] for i in range(0, len(order), self.R)]

    def fill(self, m, tenants):
        """Expand the keys of `tenants` (at most R) that hold no slot, evicting the least recently used tenants outside
        them, with one launch for the bootstrap keys and one for the key-switch keys; mark the round's tenants most
        recently used, in tenant order; then point the machine's key lists at the round's slots."""
        thr = m.thread
        missing = [t for t in tenants if t not in self.lru]
        if missing:
            keep = set(tenants)
            victims = [t for t in self.lru if t not in keep]
            slots = []
            for _ in missing:
                if self.slots < self.R:
                    in_size, t_, base = self.keys[0].ks_b.shape
                    slots.append((thr.mk_bk_slot(m.params.in_out_params.size),
                                  thr.empty((in_size, t_, base, m.params.in_out_params.size), torch.int32)))
                    self.slots += 1
                else:
                    slots.append(self.lru.pop(victims.pop(0)))
            seeds = numpy.stack([self.keys[t].seed for t in missing])
            thr.mk_bk_expand(seeds, [self.keys[t].bk_body for t in missing], [s[0] for s in slots], m.params)
            thr.mk_ks_expand(seeds, [s[1] for s in slots])
            for t, slot in zip(missing, slots):
                self.lru[t] = slot
        for t in sorted(tenants):                     # the round's tenants become the most recently used
            self.lru.move_to_end(t)
        first = self.lru[tenants[0]]
        m._bk_ints = [self.lru.get(t, first)[0] for t in range(m.tenants)]
        m._ks = [(self.lru.get(t, first)[1], self.keys[t].ks_b, self.ks_cv[self.keys[t].ks_variance])
                 for t in range(m.tenants)]


class MultiKeyVirtualMachine:
    """Executes gates, LUTs, tree LUTs, packing, expansion and index lookups on the ciphertexts of several cloud keys at
    once.

    Every operand is a list aligned with `cloud_keys`: entry t holds tenant t's ciphertexts (of any shape, broadcast per
    tenant as VirtualMachine does), or None when tenant t has no work, in which case all its operands must be None.
    The result is a list aligned the same way (None for idle tenants).

    With `resident_tenants=R` every key is a CompressedCloudKey with its bodies on the machine's device, and at most R
    tenants hold expanded keys at a time (DESIGN.md section 19); the results are the same.

    .. method:: gate_<operator>(*operand_lists, dest=None)
    """

    def __init__(self, thread, cloud_keys, perf_params: PerformanceParameters = None, resident_tenants=None):
        cloud_keys = list(cloud_keys)
        if not cloud_keys:
            raise ValueError('a multi-key machine needs at least one cloud key')
        self._pool = None
        if resident_tenants is not None:
            self._init_pool(thread, cloud_keys, perf_params, resident_tenants)
            return
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

    def _init_pool(self, thread, keys, perf_params, R):
        if isinstance(R, bool) or not isinstance(R, (int, numpy.integer)):
            raise TypeError('resident_tenants must be an int, got %s' % type(R).__name__)
        if R < 1:
            raise ValueError('resident_tenants must be at least 1, got %d' % R)
        for t, key in enumerate(keys):
            if not isinstance(key, CompressedCloudKey):
                raise TypeError('tenant %d: a multi-key machine with resident_tenants takes CompressedCloudKey objects '
                                '(ctx.load_compressed_cloud_key), got %s' % (t, type(key).__name__))
        params = keys[0].params
        pp = (perf_params if perf_params is not None else PerformanceParameters(params)).for_device(thread.device_params)
        n = params.in_out_params.size
        for t, key in enumerate(keys):
            if key.params != params:
                raise ValueError('tenant %d: the cloud key was made for other parameters than tenant 0\'s' % t)
            if key.bk_body.shape[0] != n:
                raise ValueError('tenant %d: multi-bit bootstrap keys are not supported by the multi-key machine' % t)
            if not pp.single_kernel_bootstrap or not fused_kernel_supported(params.tgsw_params):
                raise ValueError('tenant %d: the multi-key machine runs the fused bootstrap only (single_kernel_bootstrap=True, '
                                 'tlwe_mask_size=1)' % t)
            if key.bk_body.device != thread.device or key.ks_b.device != thread.device:
                raise ValueError('tenant %d: the compressed key\'s bodies are on %s, not on the machine\'s device %s'
                                 % (t, key.bk_body.device, thread.device))
        self.thread = thread
        self.params = params
        self.cloud_keys = keys
        self.perf_params = pp
        self._bk_ints = self._ks = None        # the keys of the current round (_SlotPool.fill)
        self._pool = _SlotPool(keys, int(R))

    @property
    def tenants(self):
        return len(self.cloud_keys)

    @property
    def resident(self):
        """The tenants whose keys are expanded on the device, least recently used first (resident_tenants mode; every
        tenant otherwise)."""
        return list(range(self.tenants)) if self._pool is None else list(self._pool.lru)

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

    def _concat(self, ops, active, shapes):
        parts = [_expand(ops[t], shapes[t]) for t in active]
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

    def _columns(self, cols, active, shapes, counts, dest_lists, single):
        """Per tenant, its views of several results (a, b, cv) of the whole batch (the outputs of a table, the columns
        of a lookup), or copies into its list of `dest_lists`: one array when `single`, else a list."""
        res = [self._results(c, active, shapes, counts, None if dest_lists is None else
                             [None if d is None else d[j] for d in dest_lists]) for j, c in enumerate(cols)]
        out = [None] * self.tenants
        for t in active:
            out[t] = res[0][t] if single else [r[t] for r in res]
        return out

    # --- gates ---------------------------------------------------------------------------------
    @_in_rounds(('a', 'b'), ('dest',))
    def _binary(self, name, a, b, dest):
        active, shapes = self._active((a, b), dest)
        if not active:
            return [None] * self.tenants
        num, den, sa, sb = _BINARY_GATES[name]
        counts = self._counts(active, shapes)
        ext = self.thread.mk_bootstrap_extract(self._concat(a, active, shapes), self._concat(b, active, shapes),
                                               phase_to_t32(num, den), sa, sb, MU, self._bk_ints, counts)
        return self._results(self._keyswitch(counts, ext), active, shapes, counts, dest)

    @_in_rounds(('a', 'b', 'c'), ('dest',))
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
    def _tenant_tables(self, tables, active):
        """A list of per-tenant LookupTables: the table of tenant 0's kind, after checking that every active tenant has
        one and that they share bits, log2_outputs and out."""
        if len(tables) != self.tenants:
            raise ValueError('tables must be one LookupTable or a list of %d, one per tenant' % self.tenants)
        ref = None
        for t in active:
            table = tables[t]
            if not isinstance(table, LookupTable):
                raise TypeError('tenant %d: a LookupTable is needed (vm.make_lut), got %s' % (t, type(table).__name__))
            if table.batch_shape:
                raise ValueError('tenant %d: the multi-key machine takes one table per tenant, not one per ciphertext' % t)
            if ref is None:
                ref = table
            elif (table.bits, table.log2_outputs, table.out) != (ref.bits, ref.log2_outputs, ref.out):
                raise ValueError('tenant %d: the tables must share bits, log2_outputs and out (%s, got %s)'
                                 % (t, (ref.bits, ref.log2_outputs, ref.out), (table.bits, table.log2_outputs, table.out)))
        return ref

    @_in_rounds(('xs', 'ys'), ('table', 'dest'))
    def lut(self, table, xs, ys=None, shift=0, dest=None):
        """f(x), or f(x * 2^shift + y), for every tenant's ciphertexts with one LookupTable (VirtualMachine.make_lut)
        shared by all tenants, or a list of one table per tenant (None for idle tenants), all with the same bits,
        log2_outputs and out.  Entry t of the result is one ciphertext array, or a list of 2^L of them for a table with
        several outputs.  ValueError for a configuration without enough noise margin (lut.check_noise), for tables
        with one entry per ciphertext and for per-tenant tables that differ in bits, log2_outputs or out."""
        if isinstance(table, (list, tuple)):
            tables = list(table)
            operand_lists = (xs,) if ys is None else (xs, ys)
            active, _ = self._active(operand_lists, None)
            table = self._tenant_tables(tables, active)
            if table is None:
                return [None] * self.tenants
            return self._lut(table, xs, ys, shift, dest, tables)
        if table.batch_shape:
            raise ValueError('the multi-key machine takes one table for every ciphertext, not one per ciphertext')
        return self._lut(table, xs, ys, shift, dest, None)

    def _lut(self, table, xs, ys, shift, dest, tables):
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
        p = self.params
        sh = None if ys is None else shift
        _check_config(table.bits, L, sh)
        _check_margin(_sigma(p.in_out_params, p.tgsw_params, p.ks_decomp_length, p.ks_log2_base, L, sh), table.bits, L, sh)
        out = [None] * self.tenants
        if not active:
            return out
        counts = self._counts(active, shapes)
        p1 = self._concat(xs, active, shapes)
        p2 = self._concat(ys, active, shapes) if ys is not None else None
        s1 = 1 << shift if ys is not None else 1
        tv = table.tv
        if tables is not None:      # one test vector per ciphertext: its tenant's
            tv = torch.cat([tables[t].tv.reshape(1, -1).expand(counts[t], -1) for t in active])
        keys = TenantKeys(self.thread, counts, self._bk_ints, self._ks)
        ea, eb = keys.bootstrap_lut_extract(p1, p2, s1, tv, L)
        ra, rb, rcv = keys.keyswitch((ea, eb), per=K, want_cv=True)
        # sample j of ciphertext c is row c * K + j: one contiguous block per output
        total = rb.numel() // K
        ra = ra.reshape(total, K, -1).transpose(0, 1).contiguous()
        rb = rb.reshape(total, K).t().contiguous()
        rcv = rcv.reshape(total, K).t().contiguous()
        return self._columns([(ra[j], rb[j], rcv[j]) for j in range(K)], active, shapes, counts, dest_lists, K == 1)

    # --- per-tenant extras (DESIGN.md section 18) --------------------------------------------------
    def _tenant_objects(self, objs, active, cls, what, hint=''):
        """Check a list of per-tenant objects (keys, compact ciphertexts, indices): aligned with the tenants, an
        instance of `cls` made for this machine's parameters for every active tenant."""
        if not isinstance(objs, (list, tuple)) or len(objs) != self.tenants:
            raise ValueError('%s must be a list of %d entries, one per tenant' % (what, self.tenants))
        for t in active:
            if not isinstance(objs[t], cls):
                raise TypeError('tenant %d: %s needs a %s%s, got %s' % (t, what, cls.__name__, hint, type(objs[t]).__name__))
            if objs[t].params != self.params:
                raise ValueError('tenant %d: the %s was made for other parameters than the cloud keys' % (t, what))
        return list(objs)

    def _per_tenant(self, dest, active, K, what):
        """dest as a list of lists of K results (None for idle tenants)."""
        if dest is None:
            return None
        if not isinstance(dest, (list, tuple)) or len(dest) != self.tenants:
            raise ValueError('dest must be a list of %d entries, one per tenant' % self.tenants)
        out = [None if d is None else ([d] if isinstance(d, LweSampleArray) else list(d)) for d in dest]
        active_set = set(active)
        for t in range(self.tenants):
            if (t in active_set) != (out[t] is not None):
                raise ValueError('tenant %d: a destination is needed exactly for a tenant with operands' % t)
            if out[t] is not None and len(out[t]) != K:
                raise ValueError('tenant %d: %s writes %d results, got %d' % (t, what, K, len(out[t])))
        return out

    @_in_rounds(('digits',), ('tree_keys', 'dest'))
    def lut_tree(self, tree_keys, table, digits, dest=None):
        """f(d_{D-1}, ..., d_0) for every tenant (VirtualMachine.lut_tree): `digits` is a list of D operand lists
        (highest digit first), `tree_keys` the list of the tenants' NuFHETreeKeys (None for idle tenants), `table` one
        TreeLookupTable shared by all tenants.  Every level runs once over the concatenated batch of all tenants.  Entry
        t of the result is one ciphertext array, or a list of F for a table of F functions."""
        if not isinstance(table, TreeLookupTable):
            raise TypeError('lut_tree needs a TreeLookupTable (vm.make_tree_lut), got %s' % type(table).__name__)
        if table.params != self.params or table.multi_bit != 1:
            raise ValueError('the table was made for other parameters or another kind of bootstrap key')
        digits = list(digits)
        if len(digits) != table.digits:
            raise ValueError('the table takes %d digits, got %d' % (table.digits, len(digits)))
        F = table.functions
        active, shapes = self._active(digits, None)
        tree_keys = self._tenant_objects(tree_keys, active, NuFHETreeKey, 'tree key',
                                         ' (ctx.make_cloud_key(sk, tree_key=True))')
        dest_lists = self._per_tenant(dest, active, F, 'a table of %d functions' % F)
        for t in active:
            for d in digits:
                if tuple(d[t].shape) != tuple(digits[0][t].shape):
                    raise ValueError('tenant %d: all digits must have one shape, got %s and %s'
                                     % (t, tuple(digits[0][t].shape), tuple(d[t].shape)))
            if dest_lists is not None:
                for r in dest_lists[t]:
                    check_shape(r, *[d[t] for d in digits])
                shapes[t] = tuple(dest_lists[t][0].shape)
        out = [None] * self.tenants
        if not active:
            return out
        thr = self.thread
        counts = self._counts(active, shapes)
        keys = TenantKeys(thr, [counts[t] for t in active], [self._bk_ints[t] for t in active],
                          [self._ks[t] for t in active], planes=[tree_keys[t].planes(thr) for t in active])
        flat = [self._concat(d, active, shapes) for d in reversed(digits)]        # d_0 first
        out_a, out_b = tree_lut.evaluate(keys, table, flat)
        # function f of every tenant: views of one (F, B) allocation
        out_a, out_b = out_a.transpose(0, 1).contiguous(), out_b.t().contiguous()
        variance = tree_lut.output_variance(table.params, table.bits, table.digits)
        out_cv = thr.empty((F, sum(counts)), torch.float32).fill_(float(variance))
        return self._columns([(out_a[f], out_b[f], out_cv[f]) for f in range(F)], active, shapes, counts, dest_lists,
                             table.single)

    def pack(self, packing_keys, results_list):
        """Pack every tenant's results (VirtualMachine.pack) with its NuFHEPackingKey: a list of PackedLweSampleArrays
        (None for idle tenants), each byte-identical to the tenant's own vm.pack.  Each tenant's results start at a
        group boundary, so a group never mixes tenants; the rows that pad a tenant's last group are zero, which packs
        exactly as an empty slot.  The MAC of all groups runs in one launch per pass, each group with its tenant's key."""
        active, shapes = self._active((results_list,), None)
        packing_keys = self._tenant_objects(packing_keys, active, NuFHEPackingKey, 'packing key')
        for t in active:
            if results_list[t].params != self.params.in_out_params:
                raise ValueError('tenant %d: the ciphertexts do not have the LWE parameters of the packing key' % t)
        out = [None] * self.tenants
        if not active:
            return out
        thr = self.thread
        n, N = self.params.in_out_params.size, self.params.tgsw_params.tlwe_params.polynomial_degree
        parts = [(results_list[t].a.reshape(-1, n), results_list[t].b.reshape(-1)) for t in active]
        groups = [-(-b.shape[0] // N) for a, b in parts]
        keys = TenantKeys(thr, groups, spectra=[packing_keys[t].spectra(thr) for t in active])
        data = packing.pack_groups(thr, self.params, keys, parts)
        g0 = 0
        for t, g in zip(active, groups):
            out[t] = PackedLweSampleArray(self.params, shapes[t], data[g0:g0 + g])
            g0 += g
        return out

    @_in_rounds(('compacts',))
    def expand(self, compacts):
        """The LweSampleArrays of every tenant's compact ciphertexts (VirtualMachine.expand): one extraction over all
        tenants' groups, then one multi-key key switch, a few groups per pass (compact.PASS_BYTES).  A list aligned with
        the tenants (None for idle tenants)."""
        if not isinstance(compacts, (list, tuple)) or len(compacts) != self.tenants:
            raise ValueError('compacts must be a list of %d entries, one per tenant' % self.tenants)
        active = [t for t in range(self.tenants) if compacts[t] is not None]
        compacts = self._tenant_objects(compacts, active, CompactLweSampleArray, 'compact ciphertext')
        out = [None] * self.tenants
        if not active:
            return out
        thr = self.thread
        shapes = {t: compacts[t].shape for t in active}
        counts = self._counts(active, shapes)
        B = sum(counts)
        res = (thr.empty((B, self.params.in_out_params.size), torch.int32), thr.empty((B,), torch.int32),
               thr.empty((B,), torch.float32))
        keys = TenantKeys(thr, [counts[t] for t in active], kss=[self._ks[t] for t in active])
        compact.expand_groups(thr, self.params, keys, [compacts[t] for t in active], res)
        return self._results(res, active, shapes, counts, None)

    @_in_rounds(('indexes',), ('table', 'dest'))
    def lookup(self, indexes, table, dest=None):
        """table[idx] for every tenant's EncryptedIndexArray (VirtualMachine.lookup): `table` is one IndexTable shared by
        all tenants, or a list with one EncryptedIndexTable per tenant (None for an idle tenant; DESIGN.md section 20)
        that share m, W and out.  The queries of all tenants go through one CMux tree and rotation per pass, the level
        that first reads a table taking each query's own table, then one multi-key key switch.  Entry t of the result is
        one ciphertext array of the tenant's index shape, or a list of W for a table of W columns."""
        per_tenant = isinstance(table, (list, tuple))
        if not per_tenant and not isinstance(table, IndexTable):
            raise TypeError('lookup needs an IndexTable (vm.make_index_table) or a list of EncryptedIndexTables, got %s'
                            % type(table).__name__)
        if not isinstance(indexes, (list, tuple)) or len(indexes) != self.tenants:
            raise ValueError('indexes must be a list of %d entries, one per tenant' % self.tenants)
        active = [t for t in range(self.tenants) if indexes[t] is not None]
        indexes = self._tenant_objects(indexes, active, EncryptedIndexArray, 'encrypted index',
                                       ' (decompress() a compressed one first)')
        if per_tenant:
            tables = self._tenant_objects(table, active, EncryptedIndexTable, 'encrypted table',
                                          ' (ctx.encrypt_table or vm.make_encrypted_table)')
            ref = tables[active[0]] if active else None
            for t in active:
                if (tables[t].bits, tables[t].columns, tables[t].single) != (ref.bits, ref.columns, ref.single):
                    raise ValueError('tenant %d: the tables of one call share m = %d and W = %d, got m = %d, W = %d'
                                     % (t, ref.bits, ref.columns, tables[t].bits, tables[t].columns))
        else:
            if table.params != self.params:
                raise ValueError('the table was made for other parameters than the cloud keys')
            tables, ref = None, table
        out = [None] * self.tenants
        if not active:
            return out
        for t in active:
            if indexes[t].bits != ref.bits:
                raise ValueError('tenant %d: the table takes %d-bit indices, got %d bits' % (t, ref.bits, indexes[t].bits))
        m, W = ref.bits, ref.columns
        dest_lists = self._per_tenant(dest, active, W, 'a table of %d columns' % W)
        for t in active:
            if dest_lists is not None and any(tuple(d.shape) != indexes[t].shape for d in dest_lists[t]):
                raise ValueError('tenant %d: lookup writes %d results of shape %s' % (t, W, indexes[t].shape))
        thr = self.thread
        n = self.params.in_out_params.size
        shapes = {t: indexes[t].shape for t in active}
        all_counts = self._counts(active, shapes)
        counts = [all_counts[t] for t in active]
        B = sum(counts)
        sels = [indexes[t].samples.reshape(c, m, 2, 2, 2, index_lookup.N) for t, c in zip(active, counts)]
        keys = TenantKeys(thr, counts, kss=[self._ks[t] for t in active])
        # column w of query q (of the concatenated batch) at row w B + q
        res_a, res_b = thr.empty((W * B, n), torch.int32), thr.empty((W * B,), torch.int32)
        for q0, q1, a, b in index_lookup.lookup_passes(thr, m, W, sels, None if per_tenant else table,
                                                       [tables[t] for t in active] if per_tenant else None):
            Q = q1 - q0
            pass_keys = keys.split(q0, q1)
            # rows (w, q) are column-major; the key switch wants each tenant's W c rows together, in vm.lookup's order
            lo = numpy.cumsum([0] + pass_keys.counts)
            perm = numpy.concatenate([(numpy.arange(W)[:, None] * Q + numpy.arange(lo[i], lo[i + 1])).reshape(-1)
                                      for i in range(len(pass_keys.counts))])
            sel = thr.to_device(perm)
            ra, rb, _ = pass_keys.keyswitch((a.reshape(W * Q, -1).index_select(0, sel),
                                             b.reshape(W * Q).index_select(0, sel)), per=W)
            dst = thr.to_device((perm // Q) * B + q0 + perm % Q)
            res_a.index_copy_(0, dst, ra)
            res_b.index_copy_(0, dst, rb)
        res_cv = thr.empty((W, B), torch.float32).fill_(float(index_lookup.output_variance(self.params, m)))
        if per_tenant:
            for t, lo, c in zip(active, numpy.cumsum([0] + counts), counts):
                res_cv[:, lo:lo + c] = float(tables[t].variance + index_lookup.output_variance(self.params, m))
        return self._columns([(res_a[w * B:(w + 1) * B], res_b[w * B:(w + 1) * B], res_cv[w]) for w in range(W)],
                             active, shapes, all_counts, dest_lists, ref.single)

    def _write_operands(self, what, tree_keys, tables, indexes, values):
        """Validate per-tenant writes: the active tenants (those with an index) and whether their values are LWE
        samples.  Errors name the tenant."""
        for name, lst in (('tree_keys', tree_keys), ('tables', tables), ('indexes', indexes), ('values', values)):
            if not isinstance(lst, (list, tuple)) or len(lst) != self.tenants:
                raise ValueError('%s must be a list of %d entries, one per tenant' % (name, self.tenants))
        active = [t for t in range(self.tenants) if indexes[t] is not None]
        kinds = set()
        for t in active:
            try:
                kinds.add(index_write.check_arguments(what, self.params, indexes[t], tables[t], tree_keys[t], values[t]))
            except (TypeError, ValueError) as e:
                raise type(e)('tenant %d: %s' % (t, e)) from None
            ref = tables[active[0]]
            if (tables[t].bits, tables[t].columns) != (ref.bits, ref.columns):
                raise ValueError('tenant %d: the tables of one call share m = %d and W = %d, got m = %d, W = %d'
                                 % (t, ref.bits, ref.columns, tables[t].bits, tables[t].columns))
        if len(kinds) > 1:
            raise ValueError('the values of one call are all ciphertexts or all plain integers')
        return active, bool(kinds) and kinds.pop()

    def _scatter(self, what, tree_keys, tables, indexes, values, write_variances=None):
        active, lwe = self._write_operands(what, tree_keys, tables, indexes, values)
        out = [None] * self.tenants
        if not active:
            return out
        thr = self.thread
        ref = tables[active[0]]
        m, W = ref.bits, ref.columns
        counts, a, b, variances = [], [], [], []
        for t in active:
            if tables[t].out != 'int' and write_variances is None:
                raise ValueError("tenant %d: scatter_add adds integers: it takes out='int' tables only (write overwrites "
                                 "'bool' entries)" % t)
            shape = indexes[t].shape
            B = int(numpy.prod(shape, dtype=numpy.int64))
            if lwe:
                at, bt, var = index_write.lwe_values(self.params, shape, W, values[t])
                a.append(at)
            else:
                bt, var = index_write.plain_values(thr, tables[t], shape, W, values[t]), None
            if write_variances is not None:
                var = write_variances[t]
            v = index_lookup.written_table_variance(self.params, index_write.leaf_variance(tables[t]), m, B, var,
                                                    write_variances is not None)
            try:
                index_lookup.check_table_variance(self.params, v, m, tables[t].out, tables[t].bits_out)
            except ValueError as e:
                raise ValueError('tenant %d: %s' % (t, e)) from None
            counts.append(B)
            b.append(bt)
            variances.append(v)
        accs = torch.stack([index_write.table_nodes(tables[t]) for t in active])
        keys = TenantKeys(thr, counts, planes=[tree_keys[t].planes(thr) for t in active]) if lwe else None
        sels = [indexes[t].samples.reshape(c, m, 2, 2, 2, index_lookup.N) for t, c in zip(active, counts)]
        ids = numpy.repeat(numpy.arange(len(active), dtype=numpy.uint32), counts)
        if sum(counts):
            index_write.scatter_passes(thr, self.params, keys, m, W, sels, torch.cat(a) if lwe else None, torch.cat(b),
                                       accs, ids)
        for i, t in enumerate(active):
            out[t] = index_write.finish(thr, self.params, tables[t], accs[i], variances[i])
        return out

    def scatter_add(self, tree_keys, tables, indexes, values):
        """VirtualMachine.scatter_add for every tenant with an index (None: idle), one table per tenant (the tables of a
        call share m and W): the queries of all tenants go through one tree key switch, rotation and demultiplexer per
        pass, each adding into its tenant's table.  A list of EncryptedIndexTables aligned with the tenants, each
        bit-identical to the tenant's own vm.scatter_add."""
        return self._scatter('scatter_add', tree_keys, tables, indexes, values)

    def write(self, tree_keys, tables, indexes, values):
        """VirtualMachine.write for every tenant with an index: mk.lookup of the old entries, then one scatter of
        v_q - old_q.  Each result is bit-identical to the tenant's own vm.write."""
        active, _ = self._write_operands('write', tree_keys, tables, indexes, values)
        for t in active:
            if not isinstance(tree_keys[t], NuFHETreeKey):
                raise TypeError('tenant %d: write needs a NuFHETreeKey (ctx.make_cloud_key(sk, tree_key=True)), got %s'
                                % (t, type(tree_keys[t]).__name__))
        if not active:
            return [None] * self.tenants
        if all(isinstance(tables[t], EncryptedIndexTable) for t in active):
            old = self.lookup(indexes, [tables[t] if indexes[t] is not None else None for t in range(self.tenants)])
        elif len({id(tables[t]) for t in active}) == 1:
            old = self.lookup(indexes, tables[active[0]])
        else:
            raise ValueError('write takes one EncryptedIndexTable per tenant, or one IndexTable shared by all')
        diffs, variances = [None] * self.tenants, [None] * self.tenants
        for t in active:
            diffs[t], variances[t] = index_write.differences(self.thread, tables[t], indexes[t].shape, old[t], values[t])
        return self._scatter('write', tree_keys, tables, indexes, diffs, variances)
