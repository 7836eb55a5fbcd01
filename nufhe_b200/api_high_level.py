"""High-level API (reference: nufhe/api_high_level.py): find_devices, DeviceID, Context, VirtualMachine."""
import io

import torch

from .api_low_level import (
    NuFHEParameters, NuFHESecretKey, NuFHECloudKey, encrypt, decrypt, encrypt_int, decrypt_int, empty_ciphertext)
from .lwe import LweSampleArray, lwe_copy, lwe_add_to
from .compressed import CompressedLweSampleArray, CompressedCloudKey
from .public_key import NuFHEPublicKey
from .compact import NuFHECompactPublicKey, CompactLweSampleArray, expand
from .reencrypt import NuFHEReencryptionKey, make_reencryption_key, reencrypt
from .packing import (NuFHEPackingSecretKey, NuFHEPackingKey, PackedLweSampleArray, make_packing_keys, pack,
                      decrypt_packed, decrypt_packed_int)
from .tree_lut import NuFHETreeKey, TreeLookupTable, lut_tree
from .index_lookup import (NuFHEIndexSecretKey, IndexTable, EncryptedIndexTable, encrypt_index, encrypt_table,
                           make_encrypted_table, load_encrypted_index, lookup, _check_params as check_index_params)
from .random_numbers import DeterministicRNG
from .performance import PerformanceParameters
from .computation_cache import clear_computation_cache
from .gates import result_shape, get_shape
from .engine import Engine
from . import gates, index_write


def _check_api(api):
    if api not in (None, 'CUDA', 'cuda'):
        raise ValueError("Unrecognized API: " + str(api) + " (this engine is CUDA-only)")


def _match(name, include, exclude):
    if include is not None and not any(mask in name for mask in include):
        return False
    if exclude is not None and any(mask in name for mask in exclude):
        return False
    return True


def find_devices(api=None, include_devices=None, exclude_devices=None,
                 include_platforms=None, exclude_platforms=None):
    """api_high_level.py:45-82: the CUDA devices visible to this process that pass the name filters."""
    _check_api(api)
    if not _match('NVIDIA CUDA', include_platforms, exclude_platforms):
        return []
    ids = []
    for ordinal in range(torch.cuda.device_count()):
        name = torch.cuda.get_device_name(ordinal)
        if _match(name, include_devices, exclude_devices):
            ids.append(DeviceID('CUDA', 0, ordinal, 'NVIDIA CUDA', name))
    return ids


class DeviceID:
    """A picklable device identifier (api_high_level.py:85-127)."""

    def __init__(self, api_id, platform_id, device_id, platform_name='NVIDIA CUDA', device_name=''):
        self.api_id = api_id
        self.platform_id = platform_id
        self.device_id = device_id
        self.api_name = 'CUDA'
        self.platform_name = platform_name
        self.device_name = device_name

    def get_api_and_device(self):
        return 'CUDA', self.device_id

    def __str__(self):
        return "DeviceID(api={api}, platform={pnum} ({pname}), device={dnum} ({dname}))".format(
            api=self.api_name, pnum=self.platform_id, pname=self.platform_name,
            dnum=self.device_id, dname=self.device_name)


class Context:
    """An execution environment on one GPU (api_high_level.py:130-299).

    `thread` may be a ready nufhe_b200.engine.Engine; otherwise `device_id` (a DeviceID or a CUDA
    ordinal) selects the GPU, else the first device passing the filters.  `interactive` is accepted
    and ignored."""

    def __init__(self, rng=None, thread=None, device_id=None, api=None, interactive=False,
                 include_devices=None, exclude_devices=None,
                 include_platforms=None, exclude_platforms=None):
        if rng is None:
            rng = DeterministicRNG()
        if thread is not None:
            pass
        elif device_id is not None:
            ordinal = device_id.device_id if isinstance(device_id, DeviceID) else int(device_id)
            thread = Engine(ordinal)
        else:
            _check_api(api)
            if not torch.cuda.is_available():
                raise RuntimeError("nufhe_b200 needs a CUDA device; there is no CPU fallback")
            devices = find_devices(
                api=api, include_devices=include_devices, exclude_devices=exclude_devices,
                include_platforms=include_platforms, exclude_platforms=exclude_platforms)
            if len(devices) == 0:
                raise ValueError("No devices satisfying the given filters were found")
            thread = Engine(devices[0].device_id)
        self.rng = rng
        self.thread = thread

    def __del__(self):
        if hasattr(self, 'thread'):
            clear_computation_cache(self.thread)

    def make_secret_key(self, **params):
        return NuFHESecretKey.from_rng(self.thread, NuFHEParameters(**params), self.rng)

    def make_cloud_key(self, secret_key: NuFHESecretKey, compressed=False, tree_key=False, multi_bit=1,
                       index_key=False, compact_public_key=False):
        """compressed=True returns a CompressedCloudKey (about 12 times smaller to store or send); its `decompress()`
        gives the NuFHECloudKey that make_virtual_machine takes.  tree_key=True returns (cloud key, NuFHETreeKey), the
        key of VirtualMachine.lut_tree; its draws follow all of the cloud key's, so the cloud key is the same either
        way.  multi_bit=2 gives the cloud key a MultiBitBootstrapKey (key bits two at a time: half the CMux steps per
        bootstrap, about 3x the key rows and more noise; DESIGN.md section 14); ValueError for parameters it cannot
        take (tlwe_mask_size = 2, an odd LWE dimension) and for multi_bit outside {1, 2}.
        index_key=True also returns the NuFHEIndexSecretKey that encrypts indices for VirtualMachine.lookup; it draws
        nothing.  With several extras the order is (cloud key, tree key, index key, compact public key).  ValueError for
        tlwe_mask_size != 1.
        compact_public_key=True also returns a NuFHECompactPublicKey (about 5 KB; DESIGN.md section 16): whoever holds it
        encrypts up to 1024 messages per 4 KB ciphertext, which `VirtualMachine.expand` turns into LWE samples under this
        cloud key.  Its draws follow all the other keys', so those are the same either way."""
        if index_key:
            check_index_params(secret_key.params)
        cls = CompressedCloudKey if compressed else NuFHECloudKey
        cloud_key, tgsw_key = cls.from_rng_with_tgsw_key(self.thread, secret_key.params, self.rng, secret_key,
                                                         multi_bit=multi_bit)
        out = [cloud_key]
        if tree_key:
            out.append(NuFHETreeKey.from_secret_key(self.thread, self.rng, secret_key, tgsw_key))
        if index_key:
            out.append(NuFHEIndexSecretKey.from_tgsw_key(secret_key.params, tgsw_key))
        if compact_public_key:
            out.append(NuFHECompactPublicKey.from_tgsw_key(self.thread, self.rng, secret_key.params, tgsw_key))
        return out[0] if len(out) == 1 else tuple(out)

    def encrypt_index(self, index_key: NuFHEIndexSecretKey, values, bits, compressed=False):
        """Encrypted indices 0 <= v < 2^bits (bits = 1..20) for VirtualMachine.lookup: one TGSW selector per bit,
        32 KB per bit (an EncryptedIndexArray), or 16 KB per bit with compressed=True (a CompressedEncryptedIndexArray,
        `decompress()` to compute).  ValueError for bits or values out of range."""
        return encrypt_index(self.thread, self.rng, index_key, values, bits, compressed=compressed)

    def encrypt_table(self, key, table, out='int', bits=None):
        """An EncryptedIndexTable of `table` (shape (2^m,) or (W, 2^m), as make_index_table) for VirtualMachine.lookup:
        the server stores it and reads it by encrypted index without learning any entry.  `key` is a
        NuFHECompactPublicKey (whoever holds it can upload a table) or the owner's NuFHEIndexSecretKey; 4 bytes per
        entry.  TypeError for any other key, ValueError for a table or bit count out of range."""
        return encrypt_table(self.thread, self.rng, key, table, out=out, bits=bits)

    def make_reencryption_key(self, secret_key: NuFHESecretKey, compact_public_key: NuFHECompactPublicKey):
        """The NuFHEReencryptionKey (8 KB; DESIGN.md section 22) with which a server's `VirtualMachine.reencrypt` moves
        ciphertexts under `secret_key` (the sender's) to the owner of `compact_public_key` (the recipient's), without
        decrypting them.  Anyone holding both the key and the recipient's secret key recovers the sender's secret key:
        the server must never give the key to the recipient (reencrypt.make_reencryption_key has the whole trust
        model).  TypeError for other key types, ValueError for keys of different parameters."""
        return make_reencryption_key(self.thread, self.rng, secret_key, compact_public_key)

    def make_public_key(self, secret_key: NuFHESecretKey):
        """A NuFHEPublicKey: whoever holds it can encrypt (`encrypt`, `encrypt_int`) but not decrypt."""
        return NuFHEPublicKey.from_secret_key(self.thread, self.rng, secret_key)

    def make_packing_keys(self, secret_key: NuFHESecretKey):
        """(NuFHEPackingSecretKey, NuFHEPackingKey): the client keeps the first to decrypt packed results, the server
        takes the second for `VirtualMachine.pack`."""
        return make_packing_keys(self.thread, self.rng, secret_key)

    def make_key_pair(self, **params):
        secret_key = self.make_secret_key(**params)
        cloud_key = self.make_cloud_key(secret_key)
        return secret_key, cloud_key

    def encrypt(self, key, message, compressed=False):
        """`key` is a NuFHESecretKey, a NuFHEPublicKey or a NuFHECompactPublicKey.  compressed=True (secret key only)
        returns a CompressedLweSampleArray (a seed and the bodies; `decompress()` to compute).  A compact public key
        returns a CompactLweSampleArray (`VirtualMachine.expand` to compute)."""
        return encrypt(self.thread, self.rng, key, message, compressed=compressed)

    def decrypt(self, secret_key, ciphertext):
        """An LweSampleArray with its NuFHESecretKey, or a PackedLweSampleArray with its NuFHEPackingSecretKey
        (TypeError for any other pairing)."""
        if isinstance(secret_key, NuFHEPackingSecretKey) or isinstance(ciphertext, PackedLweSampleArray):
            return decrypt_packed(self.thread, secret_key, ciphertext)
        return decrypt(self.thread, secret_key, ciphertext)

    def encrypt_int(self, key, values, bits, compressed=False):
        """Integers in [0, 2^bits), bits = 1..3, for lookup tables (VirtualMachine.lut); `key` as for encrypt()."""
        return encrypt_int(self.thread, self.rng, key, values, bits, compressed=compressed)

    def decrypt_int(self, secret_key, ciphertext, bits):
        """As for decrypt(): a packed array goes with its NuFHEPackingSecretKey."""
        if isinstance(secret_key, NuFHEPackingSecretKey) or isinstance(ciphertext, PackedLweSampleArray):
            return decrypt_packed_int(self.thread, secret_key, ciphertext, bits)
        return decrypt_int(self.thread, secret_key, ciphertext, bits)

    def make_virtual_machine(self, cloud_key: NuFHECloudKey, perf_params: PerformanceParameters = None):
        return VirtualMachine(self.thread, cloud_key, perf_params=perf_params)

    def make_multi_key_machine(self, cloud_keys, perf_params: PerformanceParameters = None, resident_tenants=None):
        """A MultiKeyVirtualMachine (nufhe_b200/multikey.py) for the list of cloud keys `cloud_keys`, one per tenant:
        its gates and LUTs take one operand list aligned with it and bootstrap every tenant's ciphertexts in one launch,
        bit-identical to each tenant's own VirtualMachine.  TypeError for anything but NuFHECloudKey objects, ValueError
        for keys of different parameters, multi-bit keys, single_kernel_bootstrap=False and keys the fused FP64 step
        cannot run.
        resident_tenants=R (an int >= 1) takes CompressedCloudKey objects with their bodies on this context's device
        (load_compressed_cloud_key) instead, and keeps at most R of them expanded on the device, about 164 MB each
        (DESIGN.md section 19): an operation on more active tenants runs in rounds of at most R, with the same results.
        TypeError for anything but CompressedCloudKey objects, ValueError for R < 1 and for the keys refused above."""
        from .multikey import MultiKeyVirtualMachine
        return MultiKeyVirtualMachine(self.thread, cloud_keys, perf_params=perf_params, resident_tenants=resident_tenants)

    def load_ciphertext(self, file_or_bytestring):
        if isinstance(file_or_bytestring, bytes):
            return LweSampleArray.loads(file_or_bytestring, self.thread)
        return LweSampleArray.load(file_or_bytestring, self.thread)

    def load_compressed_ciphertext(self, file_or_bytestring):
        if isinstance(file_or_bytestring, bytes):
            return CompressedLweSampleArray.loads(file_or_bytestring, self.thread)
        return CompressedLweSampleArray.load(file_or_bytestring, self.thread)

    def load_compressed_cloud_key(self, file_or_bytestring):
        if isinstance(file_or_bytestring, bytes):
            return CompressedCloudKey.loads(file_or_bytestring, self.thread)
        return CompressedCloudKey.load(file_or_bytestring, self.thread)

    def load_public_key(self, file_or_bytestring):
        if isinstance(file_or_bytestring, bytes):
            return NuFHEPublicKey.loads(file_or_bytestring, self.thread)
        return NuFHEPublicKey.load(file_or_bytestring, self.thread)

    def load_compact_public_key(self, file_or_bytestring):
        if isinstance(file_or_bytestring, bytes):
            return NuFHECompactPublicKey.loads(file_or_bytestring, self.thread)
        return NuFHECompactPublicKey.load(file_or_bytestring, self.thread)

    def load_compact_ciphertext(self, file_or_bytestring):
        if isinstance(file_or_bytestring, bytes):
            return CompactLweSampleArray.loads(file_or_bytestring, self.thread)
        return CompactLweSampleArray.load(file_or_bytestring, self.thread)

    def load_reencryption_key(self, file_or_bytestring):
        if isinstance(file_or_bytestring, bytes):
            return NuFHEReencryptionKey.loads(file_or_bytestring, self.thread)
        return NuFHEReencryptionKey.load(file_or_bytestring, self.thread)

    def load_packed_ciphertext(self, file_or_bytestring):
        if isinstance(file_or_bytestring, bytes):
            return PackedLweSampleArray.loads(file_or_bytestring, self.thread)
        return PackedLweSampleArray.load(file_or_bytestring, self.thread)

    def load_packing_key(self, file_or_bytestring):
        if isinstance(file_or_bytestring, bytes):
            return NuFHEPackingKey.loads(file_or_bytestring, self.thread)
        return NuFHEPackingKey.load(file_or_bytestring, self.thread)

    def load_packing_secret_key(self, file_or_bytestring):
        if isinstance(file_or_bytestring, bytes):
            return NuFHEPackingSecretKey.loads(file_or_bytestring, self.thread)
        return NuFHEPackingSecretKey.load(file_or_bytestring, self.thread)

    def load_tree_key(self, file_or_bytestring):
        if isinstance(file_or_bytestring, bytes):
            return NuFHETreeKey.loads(file_or_bytestring, self.thread)
        return NuFHETreeKey.load(file_or_bytestring, self.thread)

    def load_index_secret_key(self, file_or_bytestring):
        if isinstance(file_or_bytestring, bytes):
            return NuFHEIndexSecretKey.loads(file_or_bytestring, self.thread)
        return NuFHEIndexSecretKey.load(file_or_bytestring, self.thread)

    def load_encrypted_index(self, file_or_bytestring):
        """An EncryptedIndexArray or CompressedEncryptedIndexArray, whichever was saved."""
        if isinstance(file_or_bytestring, bytes):
            file_or_bytestring = io.BytesIO(file_or_bytestring)
        return load_encrypted_index(file_or_bytestring, self.thread)

    def load_encrypted_table(self, file_or_bytestring):
        if isinstance(file_or_bytestring, bytes):
            return EncryptedIndexTable.loads(file_or_bytestring, self.thread)
        return EncryptedIndexTable.load(file_or_bytestring, self.thread)

    def load_secret_key(self, file_or_bytestring):
        if isinstance(file_or_bytestring, bytes):
            return NuFHESecretKey.loads(file_or_bytestring, self.thread)
        return NuFHESecretKey.load(file_or_bytestring, self.thread)

    def load_cloud_key(self, file_or_bytestring):
        if isinstance(file_or_bytestring, bytes):
            return NuFHECloudKey.loads(file_or_bytestring, self.thread)
        return NuFHECloudKey.load(file_or_bytestring, self.thread)


class VirtualMachine:
    """Executes gates on ciphertexts with an encapsulated cloud key (api_high_level.py:302-363).

    .. method:: gate_<operator>(*args, dest: LweSampleArray=None)
    """

    def __init__(self, thread, cloud_key: NuFHECloudKey, perf_params: PerformanceParameters = None):
        if perf_params is None:
            perf_params = PerformanceParameters(cloud_key.params)
        perf_params = perf_params.for_device(thread.device_params)
        self.thread = thread
        self.params = cloud_key.params
        self.cloud_key = cloud_key
        self.perf_params = perf_params
        if getattr(cloud_key.bootstrap_key, 'multi_bit', 1) == 2 and not perf_params.single_kernel_bootstrap:
            raise ValueError('a multi-bit bootstrap key runs on the fused kernel only (single_kernel_bootstrap=True)')
        # lay the bootstrap key out for the fused kernel once, at VM creation rather than at the first gate
        from .tgsw import engine_format, fused_kernel_supported
        if perf_params.single_kernel_bootstrap and fused_kernel_supported(cloud_key.bootstrap_key.bk_params):
            engine_format(thread, cloud_key.bootstrap_key.tgsw)
        # and the key-switch key for the tensor-core key switch, for the same reason
        cloud_key.keyswitch_key.prepare_gemm(thread)

    def empty_ciphertext(self, shape):
        return empty_ciphertext(self.thread, self.params, shape)

    def load_ciphertext(self, file):
        return LweSampleArray.load(file, self.thread)

    def _gate(self, name, *args, dest: LweSampleArray = None):
        if dest is None:
            shapes = [get_shape(arg) for arg in args]
            dest = self.empty_ciphertext(result_shape(*shapes))
        gate_func = getattr(gates, name)
        gate_func(self.thread, self.cloud_key, dest, *args, perf_params=self.perf_params)
        return dest

    def make_lut(self, table_or_tables, bits, out='int', log2_outputs=None):
        """A lookup table on `bits`-bit integers (nufhe_b200/lut.py: LookupTable): one table of 2^bits entries, or a
        list of 2 or 4 of them for as many outputs of one bootstrap; out='bool' gives gate-compatible bits."""
        from .lut import LookupTable
        return LookupTable(self.thread, table_or_tables, bits, log2_outputs=log2_outputs, out=out)

    def lut(self, table, x, y=None, shift=0, dest=None):
        """f(x), or f(x * 2^shift + y), in one programmable bootstrap; a list of ciphertexts for a table with several
        outputs.  Raises ValueError for a configuration without enough noise margin (lut.check_noise)."""
        from .lut import bootstrap_lut
        if dest is None:
            shape = result_shape(get_shape(x), *([] if y is None else [get_shape(y)]))
            dest = [self.empty_ciphertext(shape) for _ in range(table.outputs)]
        elif isinstance(dest, LweSampleArray):
            dest = [dest]
        bootstrap_lut(self.thread, dest, self.cloud_key.bootstrap_key, self.cloud_key.keyswitch_key, table, x, y,
                      shift, perf_params=self.perf_params)
        return dest if table.outputs > 1 else dest[0]

    def make_tree_lut(self, tables, bits, digits, out='int'):
        """A lookup table on `digits` encrypted digits of `bits` bits (nufhe_b200/tree_lut.py: TreeLookupTable):
        tables of shape (F,) + (2^bits,) * digits, or (2^bits,) * digits for one function, indexed
        [f, d_{D-1}, ..., d_0].  Raises ValueError for bits outside {1, 2} and for D < 2 or above what the noise
        allows (tree_lut.max_digits: 4 at bits = 2)."""
        return TreeLookupTable(self.thread, self.params, tables, bits, digits, out=out,
                               multi_bit=getattr(self.cloud_key.bootstrap_key, 'multi_bit', 1))

    def lut_tree(self, tree_key, table, digits, dest=None):
        """f(d_{D-1}, ..., d_0) for the digit ciphertexts `digits` (highest first): one ciphertext, or a list of F for a
        table of F functions.  D levels of bootstraps; `tree_key` is the NuFHETreeKey made with this VM's cloud key
        (TypeError for anything else).  To record it with `capture`, reserve table.reserve_batch(batch)."""
        if not isinstance(tree_key, NuFHETreeKey):
            raise TypeError('lut_tree needs a NuFHETreeKey (ctx.make_cloud_key(sk, tree_key=True)), got %s'
                            % type(tree_key).__name__)
        if tree_key.params != self.params:
            raise ValueError('the tree key was made for other parameters than this virtual machine')
        if dest is None:
            shape = result_shape(*[get_shape(d) for d in digits])
            dest = [self.empty_ciphertext(shape) for _ in range(table.functions)]
        elif isinstance(dest, LweSampleArray):
            dest = [dest]
        lut_tree(self.thread, dest, self.cloud_key.bootstrap_key, self.cloud_key.keyswitch_key, tree_key, table,
                 digits, perf_params=self.perf_params)
        return dest[0] if table.single else dest

    def make_index_table(self, table, out='int', bits=None):
        """A table for encrypted-index lookups (nufhe_b200/index_lookup.py: IndexTable): shape (2^m,) or (W, 2^m),
        1 <= m <= 20, W <= 2^(10 - m) below m = 10.  out='int' encodes entries as `bits`-bit integers (for vm.lut and
        decrypt_int), out='bool' as gate bits."""
        return IndexTable(self.thread, self.params, table, out=out, bits=bits)

    def make_encrypted_table(self, tree_key: NuFHETreeKey, columns, out='int', bits=None):
        """An EncryptedIndexTable whose entries are ciphertexts this machine computed: `columns` is an LweSampleArray of
        shape (2^m,) or (W, 2^m), or a list of W of shape (2^m,), packed under the bootstrap key's GLWE key with the
        tree key (DESIGN.md section 20).  `out` / `bits` say how the entries are encoded (gate bits, or `bits`-bit
        integers).  TypeError unless tree_key is a NuFHETreeKey, ValueError for other parameters or shapes."""
        return make_encrypted_table(self.thread, self.params, tree_key, columns, out=out, bits=bits)

    def lookup(self, index, table, dest=None):
        """table[idx] for every index of the EncryptedIndexArray `index` in an IndexTable or EncryptedIndexTable: one
        ciphertext array of the index's shape, or a list of W for a table of W columns.  CMux gates only, no bootstrap
        (DESIGN.md sections 15 and 20).  TypeError for anything but an EncryptedIndexArray (decompress a compressed one
        first), ValueError for other parameters or a bit count other than the table's."""
        return lookup(self.thread, self.cloud_key.keyswitch_key, index, table, dest=dest)

    def scatter_add(self, tree_key, table, index, values):
        """T[w, idx_q] += v_q[w] for every index of the EncryptedIndexArray `index`, without learning which entries
        change (DESIGN.md section 21); repeated indexes add up.  `table` is an out='int' EncryptedIndexTable, or an
        IndexTable, which starts as the noiseless encryption of its entries.  `values` is an LweSampleArray (or a list
        of W) of the index's shape under the cloud key, with `tree_key` the NuFHETreeKey of this machine, or plain
        integers broadcast to the index's shape (tree_key=None), for counting.  Keeping sums below 2^bits is the
        caller's job, as with int_add.  Returns a new EncryptedIndexTable.  TypeError as lookup, or for anything but a
        NuFHETreeKey with LWE values; ValueError for a 'bool' table, other parameters or shapes, and for a result whose
        lookups would keep less than lut.MARGIN_SIGMAS (refresh_table it first)."""
        return index_write.scatter_add(self.thread, self.params, tree_key, table, index, values)

    def write(self, tree_key, table, index, values):
        """T[idx_q] <- v_q for every index (DESIGN.md section 21), on 'int' and 'bool' tables: scatter_add of
        v_q - lookup(idx_q).  `values` as for scatter_add (plain values are 'bool' bits for a 'bool' table); the tree
        key is needed either way.  Defined for distinct indexes: an entry that several queries name receives
        old + sum_q (v_q - old).  Errors as scatter_add."""
        return index_write.write(self.thread, self.params, self.cloud_key.keyswitch_key, tree_key, table, index, values)

    def refresh_table(self, tree_key, table):
        """The same entries with fresh noise: every entry extracted, key-switched and bootstrapped through an identity
        vm.lut (W 2^m bootstraps), then packed again with make_encrypted_table.  Every write adds noise to every entry;
        this is the way out when a write raises for lack of margin."""
        return index_write.refresh_table(self, tree_key, table)

    def int_add(self, x, y, dest=None):
        """x + y of two integer ciphertexts without a bootstrap (the caller keeps the sum below 2^bits)."""
        if dest is None:
            dest = self.empty_ciphertext(result_shape(get_shape(x), get_shape(y)))
        gates.check_shape(dest, x, y)
        lwe_copy(self.thread, dest, x)          # both nb_lwe_affine, with broadcasting and variances
        lwe_add_to(self.thread, dest, y)
        return dest

    def pack(self, packing_key: NuFHEPackingKey, ciphertexts: LweSampleArray):
        """Pack results of any shape into GLWE samples, 4 bytes per bit to download (nufhe_b200/packing.py)."""
        if packing_key.params != self.params:
            raise ValueError('the packing key was made for other parameters than this virtual machine')
        return pack(self.thread, packing_key, ciphertexts)

    def expand(self, compact: CompactLweSampleArray):
        """The LweSampleArray, of the same shape, of compact public-key ciphertexts (nufhe_b200/compact.py): sample
        extraction, then this VM's key switch, a few groups per pass.  TypeError for anything but a
        CompactLweSampleArray, ValueError for one made for other parameters."""
        if not isinstance(compact, CompactLweSampleArray):
            raise TypeError('expand needs a CompactLweSampleArray, got %s' % type(compact).__name__)
        if compact.params != self.params:
            raise ValueError('the compact ciphertexts were made for other parameters than this virtual machine')
        return expand(self.thread, self.params, self.cloud_key.keyswitch_key, compact)

    def reencrypt(self, rekey: NuFHEReencryptionKey, ciphertexts: LweSampleArray, dest: LweSampleArray = None):
        """The LweSampleArray, of the same shape and under this machine's cloud key, of `ciphertexts` under the sender's
        key of the NuFHEReencryptionKey `rekey` (made for this machine's owner; nufhe_b200/reencrypt.py).  Its variances
        are the input's plus reencrypt.reencrypt_variance and the key switch's.  TypeError for other types, ValueError for a
        key of other parameters, ciphertexts of another LWE dimension, and inputs whose recorded variance is above
        reencrypt.MAX_INPUT_VARIANCE (bootstrap them first)."""
        return reencrypt(self.thread, self.params, self.cloud_key.keyswitch_key, rekey, ciphertexts, dest)

    def capture(self, circuit, reserve_batch=None):
        """Record `circuit()` -- any sequence of this VM's gates on device-resident ciphertexts -- into a CUDA graph;
        returns a `GateGraph` whose `replay()` re-runs the whole circuit with one launch (nufhe_b200/graph.py).
        A LUT with 2^L outputs key-switches B * 2^L samples: size `reserve_batch` for that."""
        from .graph import GateGraph
        return GateGraph(self.thread, circuit, reserve_batch=reserve_batch)

    def __getattr__(self, name):
        if name.startswith('gate_'):
            return lambda *args, **kwds: self._gate(name, *args, **kwds)
        raise AttributeError(name)
