"""ctypes binding of libnufhe_b200.so (C ABI: include/nufhe_b200.h).

There is no CPU fallback: if the shared library is missing or a call fails, an exception is raised.
Status codes map to the exception types the reference raises for the same situation
(SURVEY.md section 8b): NB_EINVAL / NB_EUNSUPPORTED -> ValueError, NB_ECUDA -> RuntimeError.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# NUFHE_B200_LIB lets a developer point at an experimental build of the same ABI (tools/ only)
LIB_PATH = os.environ.get('NUFHE_B200_LIB') or os.path.join(_HERE, 'csrc', 'libnufhe_b200.so')

NB_OK, NB_EINVAL, NB_EUNSUPPORTED, NB_ECUDA = 0, -1, -2, -3
FF_ADD, FF_SUB, FF_MUL, FF_MUL_PREPARED, FF_PREPARE, FF_LSH, FF_LSH_CONST = range(7)

_vp = ctypes.c_void_p
_sz = ctypes.c_size_t
_i32 = ctypes.c_int32
_int = ctypes.c_int

# name -> argtypes; mirrors include/nufhe_b200.h exactly (tests/test_host_logic.py checks it against the header)
SIGNATURES = {
    'nb_ctx_create': [_int, _vp, ctypes.POINTER(_vp)],
    'nb_ctx_destroy': [_vp],
    'nb_last_error': [_vp],
    'nb_ctx_set_stream': [_vp, _vp],
    'nb_ctx_synchronize': [_vp],
    'nb_ctx_reserve': [_vp, _sz],
    'nb_build_info': [],
    'nb_ntt_forward_i32': [_vp, _vp, _vp, _sz],
    'nb_ntt_forward_u64': [_vp, _vp, _vp, _sz],
    'nb_ntt_inverse_i32': [_vp, _vp, _vp, _sz],
    'nb_ntt_inverse_u64': [_vp, _vp, _vp, _sz],
    'nb_ff_elementwise': [_vp, _int, _vp, _vp, _vp, _sz, _sz],
    'nb_bk_row_u64': [],
    'nb_bk_prepare': [_vp, _vp, _vp, _sz],
    'nb_bk_multibit_row_u64': [],
    'nb_bk_prepare_multibit': [_vp, _vp, _vp, _sz],
    'nb_external_product': [_vp, _vp, _vp, _sz, _sz],
    'nb_blind_rotate': [_vp, _vp, _vp, _vp, _sz, _vp, _vp, _vp, _sz],
    'nb_bootstrap_extract': [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _sz, _vp, _vp, _sz],
    'nb_bootstrap_lut_extract': [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _vp, _sz, _int, _vp, _sz, _vp, _vp, _sz],
    'nb_bootstrap_extract2': [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32,
                              _vp, _sz, _vp, _vp, _sz],
    'nb_keyswitch': [_vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _vp, _sz, _sz, _int, _int, _vp, _vp, _vp, _sz],
    'nb_mk_bootstrap_extract': [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _sz, _sz, _vp, _vp, _sz],
    'nb_mk_bootstrap_extract2': [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32,
                                 _vp, _vp, _sz, _sz, _vp, _vp, _sz],
    'nb_mk_bootstrap_lut_extract': [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _vp, _sz, _int, _vp, _vp, _sz, _sz, _vp,
                                    _vp, _sz],
    'nb_mk_keyswitch': [_vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _sz, _sz, _sz, _int, _int, _vp, _vp, _vp,
                        _sz],
    'nb_mk_bootstrap_glwe_lut_extract': [_vp, _vp, _vp, _vp, _vp, _vp, _sz, _sz, _vp, _vp, _sz],
    'nb_mk_tree_keyswitch': [_vp, _vp, _vp, _vp, _sz, _sz, _int, _vp, _sz],
    'nb_mk_ntt_mac': [_vp, _vp, _vp, _vp, _sz, _vp, _sz, _sz, _sz],
    'nb_mk_bk_expand': [_vp, _vp, _vp, _vp, _sz, _sz, _int, _int, _sz],
    'nb_mk_ks_expand': [_vp, _vp, _vp, _sz, _sz, _int, _int, _sz],
    'nb_mk_slot_release': [_vp, _vp],
    'nb_ks_prepared_bytes': [],
    'nb_ks_prepare': [_vp, _vp, _vp, _vp, _sz, _sz, _int, _int, _vp],
    'nb_ks_forget': [_vp, _vp],
    'nb_lwe_affine': [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _sz, _sz],
    'nb_shift_torus_polynomial': [_vp, _vp, _vp, _vp, _sz, _sz, _int, _int, _int, _sz],
    'nb_tlwe_noiseless_trivial': [_vp, _vp, _vp, _vp, _int, _int, _sz],
    'nb_tlwe_extract_lwe_samples': [_vp, _vp, _vp, _vp, _int, _int, _sz],
    'nb_tlwe_add_to': [_vp, _vp, _vp, _sz, _vp, _vp, _sz],
    'nb_t32_to_phase': [_vp, _vp, _vp, _sz, ctypes.c_uint32],
    'nb_tgsw_decompose': [_vp, _vp, _vp, _sz, _int, _int, _i32, _int],
    'nb_tgsw_mac': [_vp, _vp, _vp, _vp, _sz, _int, _int],
    'nb_lwe_dot': [_vp, _vp, _vp, _vp, _vp, _vp, _i32, _sz, _sz],
    'nb_make_keyswitch_key': [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _sz, _int, _int, ctypes.c_float],
    'nb_seeded_uniform_i32': [_vp, _vp, ctypes.c_uint64, ctypes.c_uint64, _vp, _sz],
    'nb_pk_planes_bytes': [_sz, _sz],
    'nb_pk_prepare': [_vp, _vp, _vp, _sz, _sz, _vp],
    'nb_pk_encrypt': [_vp, _vp, _vp, _sz, _sz, _vp, ctypes.c_float, _vp, _vp, _vp, _sz],
    'nb_pack_digits': [_vp, _vp, _sz, _vp, _sz],
    'nb_ntt_mac': [_vp, _vp, _vp, _vp, _sz, _sz, _sz],
    'nb_pack_finish': [_vp, _vp, _vp, _int, _vp, _sz],
    'nb_tree_planes_bytes': [_sz, _int],
    'nb_tree_prepare': [_vp, _vp, _vp, _sz, _int, _vp],
    'nb_tree_keyswitch': [_vp, _vp, _vp, _sz, _int, _vp, _sz],
    'nb_tree_assemble': [_vp, _vp, _vp, _int, _int, _vp, _sz],
    'nb_bootstrap_glwe_lut_extract': [_vp, _vp, _vp, _vp, _vp, _sz, _vp, _vp, _sz],
    'nb_index_prepare': [_vp, _vp, _sz, _vp],
    'nb_index_cmux_level': [_vp, _vp, _sz, _vp, _sz, _vp, _sz, _sz],
    'nb_index_rotate_extract': [_vp, _vp, _sz, _vp, _sz, _int, _sz, _vp, _vp, _sz],
    'nb_index_cmux_level_indirect': [_vp, _vp, _sz, _sz, _vp, _vp, _sz, _vp, _sz, _sz],
    'nb_index_rotate_extract_indirect': [_vp, _vp, _sz, _sz, _vp, _vp, _sz, _int, _sz, _vp, _vp, _sz],
    'nb_index_write_assemble': [_vp, _vp, _vp, _int, _sz, _vp, _sz],
    'nb_index_write_rotate': [_vp, _vp, _vp, _sz, _int, _sz, _vp, _vp, _sz, _sz, _vp, _sz],
    'nb_index_demux_level': [_vp, _vp, _vp, _sz, _vp, _vp, _sz, _sz, _vp, _sz, _sz],
    'nb_compact_finish': [_vp, _vp, _vp, _vp, _vp, _int, _vp, _sz],
    'nb_compact_extract': [_vp, _vp, _int, _vp, _vp, _sz],
    'nb_reencrypt': [_vp, _vp, _vp, _sz, _int, _vp, _vp, _vp, _sz, _vp, _vp, _sz],
}
_RESTYPES = {'nb_bk_row_u64': ctypes.c_size_t, 'nb_ks_prepared_bytes': ctypes.c_size_t, 'nb_bk_multibit_row_u64': ctypes.c_size_t, 'nb_pk_planes_bytes': ctypes.c_size_t,
             'nb_tree_planes_bytes': ctypes.c_size_t, 'nb_ctx_destroy': None, 'nb_last_error': ctypes.c_char_p,
             'nb_build_info': ctypes.c_char_p}

_lib = None


def load():
    """Load the shared library (once).  Raises ImportError with build instructions if it is absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                "nufhe_b200: %s not found.  Build it with `python -c 'import __graft_entry__ as g; "
                "g.build()'` (nvcc, sm_90a).  There is no CPU fallback." % LIB_PATH)
        lib = ctypes.CDLL(LIB_PATH)
        for name, argtypes in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.argtypes = argtypes
            fn.restype = _RESTYPES.get(name, _int)
        _lib = lib
    return _lib


class NativeError(RuntimeError):
    pass


def check(ctx_handle, rc, what):
    if rc == NB_OK:
        return
    msg = load().nb_last_error(ctx_handle)
    msg = msg.decode() if msg else ''
    text = '%s failed (%d): %s' % (what, rc, msg)
    if rc in (NB_EINVAL, NB_EUNSUPPORTED):
        raise ValueError(text)
    raise NativeError(text)
