"""ctypes binding of libcpb200.so (include/cpb200.h).  Plumbing only: every computation happens in
the CUDA library.  Importing this module never touches the GPU; the first context creation does.
The library is loaded eagerly and its absence is an error -- there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, os.environ.get("CPB_LIB_NAME", "libcpb200.so"))   # CPB_LIB_NAME: development variants only

u64p = C.POINTER(C.c_uint64)
szp = C.POINTER(C.c_size_t)
u8p = C.POINTER(C.c_uint8)
vp = C.c_void_p

CPB_OK, CPB_BAD_LENGTH, CPB_BAD_PARAMS, CPB_NOT_POW2, CPB_CUDA_ERROR, CPB_NO_DEVICE, CPB_UNSUPPORTED, CPB_NULL_POINTER, CPB_INTERNAL_ERROR, CPB_NCCL_ERROR = range(10)

class SpongeMode(C.Structure):
    """cpb_sponge_mode (DuplexSpongeMode): squeezing 0 = Absorbing{index}, 1 = Squeezing{index}."""
    _fields_ = [("squeezing", C.c_int), ("index", C.c_size_t)]


modep = C.POINTER(SpongeMode)

# name -> (restype, argtypes); mirrors include/cpb200.h one to one (tests/test_abi.py checks it).
SIGNATURES = {
    "cpb_last_error": (C.c_char_p, []),
    "cpb_abi_version": (C.c_int, []),
    "cpb_version": (C.c_int, []),
    "cpb_device_count": (C.c_int, []),
    "cpb_host_register": (C.c_int, [vp, C.c_size_t]),
    "cpb_host_unregister": (C.c_int, [vp]),
    "cpb_merkle_poseidon_launch_count": (C.c_size_t, [vp, C.c_size_t]),
    "cpb_field_modulus": (C.c_int, [C.c_int, u64p]),
    "cpb_field_to_montgomery": (C.c_int, [C.c_int, C.c_int, u64p, u64p, C.c_size_t]),
    "cpb_field_from_montgomery": (C.c_int, [C.c_int, C.c_int, u64p, u64p, C.c_size_t]),
    "cpb_field_to_montgomery_dev": (C.c_int, [C.c_int, C.c_int, vp, vp, C.c_size_t, vp]),
    "cpb_field_from_montgomery_dev": (C.c_int, [C.c_int, C.c_int, vp, vp, C.c_size_t, vp]),
    "cpb_poseidon_find_ark_and_mds": (C.c_int, [C.c_int, C.c_uint64, C.c_int, C.c_int, C.c_int, C.c_int, u64p, u64p]),
    "cpb_poseidon_default_entry": (C.c_int, [C.c_int, C.c_int, C.c_int, u64p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "cpb_poseidon_ctx_create": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_uint64, u64p, u64p, C.c_int, C.POINTER(vp)]),
    "cpb_poseidon_ctx_destroy": (None, [vp]),
    "cpb_poseidon_ctx_is_sparse": (C.c_int, [vp]),
    "cpb_poseidon_ctx_field": (C.c_int, [vp]),
    "cpb_poseidon_ctx_device": (C.c_int, [vp]),
    "cpb_poseidon_permute_batch": (C.c_int, [vp, u64p, u64p, C.c_size_t]),
    "cpb_poseidon_permute_batch_dev": (C.c_int, [vp, vp, vp, C.c_size_t, vp]),
    "cpb_poseidon_crh_batch": (C.c_int, [vp, u64p, C.c_size_t, u64p, C.c_size_t]),
    "cpb_poseidon_crh_batch_dev": (C.c_int, [vp, vp, C.c_size_t, vp, C.c_size_t, vp]),
    "cpb_poseidon_sponge_batch": (C.c_int, [vp, u64p, C.c_size_t, u64p, C.c_size_t, C.c_size_t]),
    "cpb_poseidon_sponge_batch_dev": (C.c_int, [vp, vp, C.c_size_t, vp, C.c_size_t, C.c_size_t, vp]),
    "cpb_merkle_poseidon_verify_batch": (C.c_int, [vp, vp, u64p, u64p, C.c_size_t, u64p, u64p, C.c_size_t, u64p, u8p, C.c_size_t]),
    "cpb_merkle_poseidon_verify_batch_dev": (C.c_int, [vp, vp, vp, vp, C.c_size_t, vp, vp, C.c_size_t, vp, vp, C.c_size_t, vp]),
    "cpb_poseidon_crh_ragged_batch": (C.c_int, [vp, u64p, u64p, u64p, C.c_size_t]),
    "cpb_poseidon_crh_ragged_batch_dev": (C.c_int, [vp, vp, vp, vp, C.c_size_t, vp]),
    "cpb_poseidon_sponge_ragged_batch": (C.c_int, [vp, u64p, u64p, u64p, C.c_size_t, C.c_size_t]),
    "cpb_poseidon_sponge_ragged_batch_dev": (C.c_int, [vp, vp, vp, vp, C.c_size_t, C.c_size_t, vp]),
    "cpb_merkle_poseidon_build_ragged": (C.c_int, [vp, vp, u64p, u64p, C.c_size_t, u64p, u64p]),
    "cpb_merkle_poseidon_build_ragged_dev": (C.c_int, [vp, vp, vp, vp, C.c_size_t, vp, vp, vp]),
    "cpb_merkle_poseidon_verify_ragged_batch": (C.c_int, [vp, vp, u64p, u64p, u64p, u64p, u64p, C.c_size_t, u64p, u8p, C.c_size_t]),
    "cpb_merkle_poseidon_verify_ragged_batch_dev": (C.c_int, [vp, vp, vp, vp, vp, vp, vp, C.c_size_t, vp, vp, C.c_size_t, vp]),
    "cpb_poseidon_compress_batch": (C.c_int, [vp, u64p, u64p, C.c_size_t]),
    "cpb_poseidon_compress_batch_dev": (C.c_int, [vp, vp, vp, C.c_size_t, vp]),
    "cpb_poseidon_duplex_absorb": (C.c_int, [vp, u64p, modep, u64p, C.c_size_t, C.c_size_t]),
    "cpb_poseidon_duplex_absorb_dev": (C.c_int, [vp, vp, modep, vp, C.c_size_t, C.c_size_t, vp]),
    "cpb_poseidon_duplex_absorb_bytes": (C.c_int, [vp, u64p, modep, u8p, C.c_size_t, C.c_size_t, C.c_size_t]),
    "cpb_poseidon_duplex_absorb_bytes_dev": (C.c_int, [vp, vp, modep, vp, C.c_size_t, C.c_size_t, C.c_size_t, vp]),
    "cpb_poseidon_duplex_squeeze": (C.c_int, [vp, u64p, modep, u64p, C.c_size_t, C.c_int, C.c_size_t]),
    "cpb_poseidon_duplex_squeeze_dev": (C.c_int, [vp, vp, modep, vp, C.c_size_t, C.c_int, C.c_size_t, vp]),
    "cpb_poseidon_duplex_absorb_ragged": (C.c_int, [vp, u64p, modep, u64p, u64p, C.c_size_t]),
    "cpb_poseidon_duplex_absorb_ragged_dev": (C.c_int, [vp, vp, vp, vp, vp, C.c_size_t, vp]),
    "cpb_poseidon_duplex_absorb_bytes_ragged": (C.c_int, [vp, u64p, modep, u8p, u64p, C.c_size_t]),
    "cpb_poseidon_duplex_absorb_bytes_ragged_dev": (C.c_int, [vp, vp, vp, vp, vp, C.c_size_t, vp]),
    "cpb_poseidon_duplex_squeeze_ragged": (C.c_int, [vp, u64p, modep, u64p, u64p, C.c_int, C.c_size_t]),
    "cpb_poseidon_duplex_squeeze_ragged_dev": (C.c_int, [vp, vp, vp, vp, vp, C.c_int, C.c_size_t, vp]),
    "cpb_merkle_poseidon_build": (C.c_int, [vp, vp, u64p, C.c_size_t, C.c_size_t, u64p, u64p]),
    "cpb_merkle_poseidon_build_dev": (C.c_int, [vp, vp, vp, C.c_size_t, C.c_size_t, vp, vp, vp]),
    "cpb_merkle_poseidon_from_digests": (C.c_int, [vp, u64p, C.c_size_t, u64p]),
    "cpb_merkle_poseidon_from_digests_dev": (C.c_int, [vp, vp, C.c_size_t, vp, vp]),
    "cpb_merkle_poseidon_update_digests_dev": (C.c_int, [vp, vp, vp, C.c_size_t, vp, vp, C.c_size_t, vp, vp, vp]),
    "cpb_merkle_poseidon_update_dev": (C.c_int, [vp, vp, vp, vp, C.c_size_t, vp, vp, C.c_size_t, C.c_size_t, vp, vp, vp]),
    "cpb_merkle_poseidon_update_digests": (C.c_int, [vp, u64p, u64p, C.c_size_t, u64p, u64p, C.c_size_t, u64p, C.POINTER(C.c_int)]),
    "cpb_merkle_poseidon_update": (C.c_int, [vp, vp, u64p, u64p, C.c_size_t, u64p, u64p, C.c_size_t, C.c_size_t, u64p, C.POINTER(C.c_int)]),
    "cpb_pedersen_ctx_create": (C.c_int, [C.c_int, C.c_int, C.c_int, u64p, C.c_size_t, u64p, C.c_int, C.POINTER(vp)]),
    "cpb_pedersen_ctx_create_ex": (C.c_int, [C.c_int, C.c_int, C.c_int, u64p, C.c_size_t, u64p, C.c_int, C.c_int, C.POINTER(vp)]),
    "cpb_pedersen_ctx_destroy": (None, [vp]),
    "cpb_pedersen_crh_batch": (C.c_int, [vp, u8p, C.c_size_t, C.c_size_t, u64p, C.c_size_t]),
    "cpb_pedersen_crh_batch_dev": (C.c_int, [vp, vp, C.c_size_t, C.c_size_t, vp, C.c_size_t, vp]),
    "cpb_pedersen_crh_x_batch": (C.c_int, [vp, u8p, C.c_size_t, C.c_size_t, u64p, C.c_size_t]),
    "cpb_pedersen_crh_x_batch_dev": (C.c_int, [vp, vp, C.c_size_t, C.c_size_t, vp, C.c_size_t, vp]),
    "cpb_pedersen_two_to_one_batch": (C.c_int, [vp, u64p, u64p, C.c_size_t]),
    "cpb_pedersen_two_to_one_batch_dev": (C.c_int, [vp, vp, vp, C.c_size_t, vp, vp]),
    "cpb_pedersen_commit_batch": (C.c_int, [vp, u8p, C.c_size_t, C.c_size_t, u8p, u64p, C.c_size_t]),
    "cpb_pedersen_commit_batch_dev": (C.c_int, [vp, vp, C.c_size_t, C.c_size_t, vp, vp, C.c_size_t, vp]),
    "cpb_bowe_hopwood_ctx_create": (C.c_int, [C.c_int, C.c_int, C.c_int, u64p, C.c_int, C.POINTER(vp)]),
    "cpb_bowe_hopwood_ctx_destroy": (None, [vp]),
    "cpb_bowe_hopwood_crh_batch": (C.c_int, [vp, u8p, C.c_size_t, C.c_size_t, u64p, C.c_size_t]),
    "cpb_bowe_hopwood_crh_batch_dev": (C.c_int, [vp, vp, C.c_size_t, C.c_size_t, vp, C.c_size_t, vp]),
    "cpb_bowe_hopwood_two_to_one_batch": (C.c_int, [vp, u64p, u64p, C.c_size_t]),
    "cpb_bowe_hopwood_two_to_one_batch_dev": (C.c_int, [vp, vp, vp, C.c_size_t, vp, vp]),
    "cpb_bowe_hopwood_two_to_one_scratch_bytes": (C.c_size_t, [vp, C.c_size_t]),
    "cpb_merkle_pedersen_build": (C.c_int, [vp, vp, u8p, C.c_size_t, C.c_size_t, u64p, u64p]),
    "cpb_merkle_pedersen_build_dev": (C.c_int, [vp, vp, vp, C.c_size_t, C.c_size_t, C.c_size_t, vp, vp, vp, vp]),
    "cpb_merkle_pedersen_update_digests_dev": (C.c_int, [vp, vp, vp, C.c_size_t, vp, vp, C.c_size_t, vp, vp, vp]),
    "cpb_merkle_pedersen_update_dev": (C.c_int, [vp, vp, vp, vp, C.c_size_t, vp, vp, C.c_size_t, C.c_size_t, C.c_size_t, vp, vp, vp]),
    "cpb_merkle_pedersen_update_digests": (C.c_int, [vp, u64p, u64p, C.c_size_t, u64p, u64p, C.c_size_t, u64p, C.POINTER(C.c_int)]),
    "cpb_merkle_pedersen_update": (C.c_int, [vp, vp, u64p, u64p, C.c_size_t, u64p, u8p, C.c_size_t, C.c_size_t, u64p, C.POINTER(C.c_int)]),
    "cpb_merkle_mixed_build": (C.c_int, [vp, vp, u8p, C.c_size_t, C.c_size_t, u64p, u64p]),
    "cpb_merkle_mixed_build_dev": (C.c_int, [vp, vp, vp, C.c_size_t, C.c_size_t, C.c_size_t, vp, vp, vp]),
    "cpb_merkle_pedersen_verify_batch": (C.c_int, [vp, vp, u64p, u8p, C.c_size_t, u64p, u64p, C.c_size_t, u64p, u8p, C.c_size_t]),
    "cpb_merkle_pedersen_verify_batch_dev": (C.c_int, [vp, vp, vp, vp, C.c_size_t, C.c_size_t, vp, vp, C.c_size_t, vp, vp, C.c_size_t, vp]),
    "cpb_merkle_mixed_verify_batch": (C.c_int, [vp, vp, u64p, u8p, C.c_size_t, u64p, u64p, C.c_size_t, u64p, u8p, C.c_size_t]),
    "cpb_merkle_mixed_verify_batch_dev": (C.c_int, [vp, vp, vp, vp, C.c_size_t, C.c_size_t, vp, vp, C.c_size_t, vp, vp, C.c_size_t, vp]),
    "cpb_exchange_create": (C.c_int, [C.c_int, C.c_int, C.c_int, C.POINTER(vp)]),
    "cpb_exchange_destroy": (None, [vp]),
    "cpb_exchange_world": (C.c_int, [vp]),
    "cpb_exchange_rank": (C.c_int, [vp]),
    "cpb_exchange_ipc_handle": (C.c_int, [vp, u8p]),
    "cpb_exchange_connect_ipc": (C.c_int, [vp, u8p]),
    "cpb_exchange_connect_local": (C.c_int, [C.POINTER(vp), C.c_int]),
    "cpb_merkle_poseidon_build_sharded_dev": (C.c_int, [vp, vp, vp, vp, C.c_size_t, C.c_size_t, vp, vp, vp, vp]),
    "cpb_merkle_poseidon_build_sharded": (C.c_int, [vp, vp, vp, u64p, C.c_size_t, C.c_size_t, u64p, u64p, u64p]),
    "cpb_merkle_poseidon_from_digests_sharded_dev": (C.c_int, [vp, vp, vp, C.c_size_t, vp, vp, vp]),
    "cpb_merkle_mixed_build_sharded_dev": (C.c_int, [vp, vp, vp, vp, C.c_size_t, C.c_size_t, C.c_size_t, vp, vp, vp, vp]),
    "cpb_field_serialized_size": (C.c_size_t, [C.c_int]),
    "cpb_field_serialize": (C.c_int, [C.c_int, u64p, C.c_size_t, u8p]),
    "cpb_field_deserialize": (C.c_int, [C.c_int, u8p, C.c_size_t, u64p]),
    "cpb_point_serialized_size": (C.c_size_t, [C.c_int, C.c_int]),
    "cpb_point_serialize": (C.c_int, [C.c_int, u64p, C.c_size_t, C.c_int, u8p]),
    "cpb_point_deserialize": (C.c_int, [C.c_int, u8p, C.c_size_t, C.c_int, C.c_int, u64p]),
    "cpb_poseidon_config_serialize": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_uint64, u64p, u64p, u8p, C.c_size_t, szp]),
    "cpb_poseidon_config_deserialize": (C.c_int, [C.c_int, u8p, C.c_size_t, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int),
                                                  C.POINTER(C.c_int), u64p, u64p, C.c_size_t, u64p, C.c_size_t]),
    "cpb_pedersen_parameters_serialize": (C.c_int, [C.c_int, C.c_int, C.c_int, u64p, C.c_int, u8p, C.c_size_t, szp]),
    "cpb_pedersen_parameters_deserialize": (C.c_int, [C.c_int, u8p, C.c_size_t, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), u64p, C.c_size_t]),
    "cpb_path_serialize": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, u64p, u64p, C.c_size_t, C.c_uint64, u8p, C.c_size_t, szp]),
    "cpb_path_deserialize": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, u8p, C.c_size_t, u64p, u64p, C.c_size_t, szp, u64p]),
    "cpb_multipath_serialize": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_size_t, u64p, u64p, u64p, u64p, u64p, u8p, C.c_size_t, szp]),
    "cpb_multipath_deserialize": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, u8p, C.c_size_t, szp, szp, u64p, u64p, u64p, u64p, u64p,
                                            C.c_size_t, C.c_size_t]),
    "cpb_multi_create": (C.c_int, [C.c_int, C.POINTER(C.c_int), C.POINTER(vp)]),
    "cpb_multi_destroy": (None, [vp]),
    "cpb_multi_uses_nccl": (C.c_int, [vp]),
    "cpb_merkle_poseidon_build_multi": (C.c_int, [vp, C.POINTER(vp), C.POINTER(vp), u64p, C.c_size_t, C.c_size_t, u64p, u64p]),
    "cpb_te_base_ctx_create": (C.c_int, [C.c_int, u64p, C.c_int, C.POINTER(vp)]),
    "cpb_te_base_ctx_create_ex": (C.c_int, [C.c_int, u64p, C.c_int, C.POINTER(vp)]),
    "cpb_te_base_ctx_destroy": (None, [vp]),
    "cpb_te_base_mul_batch": (C.c_int, [vp, u64p, u64p, C.c_size_t]),
    "cpb_te_base_mul_batch_dev": (C.c_int, [vp, vp, vp, C.c_size_t, vp]),
    "cpb_schnorr_sign_batch": (C.c_int, [vp, u8p, u64p, u64p, u8p, u64p, u64p, u8p, C.c_size_t]),
    "cpb_schnorr_sign_batch_dev": (C.c_int, [vp, u8p, vp, vp, vp, vp, vp, vp, C.c_size_t, vp]),
    "cpb_schnorr_verify_batch": (C.c_int, [vp, u8p, u64p, u8p, u64p, u64p, u8p, C.c_size_t]),
    "cpb_schnorr_verify_batch_dev": (C.c_int, [vp, u8p, vp, vp, vp, vp, vp, C.c_size_t, vp]),
    "cpb_schnorr_randomize_public_key_batch": (C.c_int, [vp, u64p, u8p, C.c_size_t, C.c_size_t, u64p, C.c_size_t]),
    "cpb_schnorr_randomize_public_key_batch_dev": (C.c_int, [vp, vp, vp, C.c_size_t, C.c_size_t, vp, C.c_size_t, vp]),
    "cpb_schnorr_randomize_signature_batch": (C.c_int, [vp, u64p, u8p, C.c_size_t, C.c_size_t, u64p, C.c_size_t]),
    "cpb_schnorr_randomize_signature_batch_dev": (C.c_int, [vp, vp, vp, C.c_size_t, C.c_size_t, vp, C.c_size_t, vp]),
    "cpb_elgamal_encrypt_batch": (C.c_int, [vp, u64p, u64p, u64p, u64p, C.c_size_t]),
    "cpb_elgamal_encrypt_batch_dev": (C.c_int, [vp, vp, vp, vp, vp, C.c_size_t, vp]),
    "cpb_elgamal_decrypt_batch": (C.c_int, [vp, u64p, u64p, u64p, C.c_size_t]),
    "cpb_elgamal_decrypt_batch_dev": (C.c_int, [vp, vp, vp, vp, C.c_size_t, vp]),
    "cpb_blake2s_commit_batch": (C.c_int, [C.c_int, u8p, u64p, u8p, u8p, C.c_size_t]),
    "cpb_blake2s_commit_batch_dev": (C.c_int, [C.c_int, vp, vp, vp, vp, C.c_size_t, vp]),
}


class CpbError(RuntimeError):
    def __init__(self, status: int, message: str):
        super().__init__(f"cpb status {status}: {message}")
        self.status = status


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python crypto_primitives_b200/_build.py` "
            "(nvcc, sm_90a).  crypto_primitives_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)       # AttributeError if the library does not export the symbol
        fn.restype = res
        fn.argtypes = args
    return lib


lib = _load()


def check(status: int):
    if status != CPB_OK:
        raise CpbError(status, lib.cpb_last_error().decode("utf-8", "replace"))
