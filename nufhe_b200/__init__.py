"""nufhe_b200 -- an H100-native (sm_90a) engine for the gate-bootstrapping hot path of nucypher/nufhe,
behind nufhe's own API surface (nufhe/__init__.py:18-59): `import nufhe_b200 as nufhe`.

Python here is host logic only; every ciphertext operation on the path runs in hand-written CUDA
reached through the C ABI of libnufhe_b200.so (include/nufhe_b200.h).  There is no CPU fallback.
"""
from .api_low_level import (
    make_key_pair,
    encrypt,
    decrypt,
    encrypt_int,
    decrypt_int,
    empty_ciphertext,
    NuFHEParameters,
    NuFHESecretKey,
    NuFHECloudKey,
    )
from .lwe import (
    LweSampleArray,
    concatenate,
    )
from .gates import (
    gate_nand,
    gate_or,
    gate_and,
    gate_xor,
    gate_xnor,
    gate_not,
    gate_copy,
    gate_constant,
    gate_nor,
    gate_andny,
    gate_andyn,
    gate_orny,
    gate_oryn,
    gate_mux,
    )
from .lut import (
    LookupTable,
    make_test_vector,
    bootstrap_lut,
    check_noise,
    )
from .compressed import (
    CompressedLweSampleArray,
    CompressedCloudKey,
    )
from .bootstrap import MultiBitBootstrapKey
from .public_key import (
    NuFHEPublicKey,
    public_key_size,
    public_encrypt,
    )
from .packing import (
    NuFHEPackingSecretKey,
    NuFHEPackingKey,
    PackedLweSampleArray,
    make_packing_keys,
    pack,
    )
from .compact import (
    NuFHECompactPublicKey,
    CompactLweSampleArray,
    compact_encrypt,
    expand,
    )
from .reencrypt import (
    NuFHEReencryptionKey,
    make_reencryption_key,
    reencrypt_variance,
    MAX_INPUT_VARIANCE,
    )
from .tree_lut import (
    NuFHETreeKey,
    TreeLookupTable,
    lut_tree,
    )
from .index_lookup import (
    NuFHEIndexSecretKey,
    EncryptedIndexArray,
    CompressedEncryptedIndexArray,
    IndexTable,
    EncryptedIndexTable,
    encrypt_index,
    encrypt_table,
    make_encrypted_table,
    lookup,
    )
from .multikey import MultiKeyVirtualMachine
from .performance import PerformanceParameters
from .random_numbers import DeterministicRNG, SecureRNG
from .computation_cache import clear_computation_cache
from .api_high_level import (
    find_devices,
    Context,
    )

__version__ = '0.1.0'
