"""ctypes binding of circl_b200/libcirclb200.so (the C ABI in include/circl_b200.h).

The library is the product; this module only loads it.  There is no CPU
fallback: a missing library or a missing GPU raises.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libcirclb200.so")

# every symbol include/circl_b200.h declares (checked by tests/test_abi.py)
SYMBOLS = {
    "cb200_init": (C.c_int, [C.c_int]),
    "cb200_init_devices": (C.c_int, [C.c_int]),
    "cb200_active_devices": (C.c_int, []),
    "cb200_shutdown": (None, []),
    "cb200_device_count": (C.c_int, []),
    "cb200_last_error": (C.c_char_p, []),
    "cb200_version": (C.c_char_p, []),
    "cb200_set_stream": (C.c_int, [C.c_void_p]),
    "cb200_release_stream": (C.c_int, [C.c_void_p]),
    "cb200_synchronize": (C.c_int, []),
    "cb200_bind_thread_to_device": (C.c_int, [C.c_int]),
    "cb200_gather_alloc": (C.c_int, [C.c_size_t, C.c_void_p, C.c_void_p]),
    "cb200_gather_free": (C.c_int, [C.c_void_p]),
    "cb200_gather_open": (C.c_int, [C.c_void_p, C.c_void_p]),
    "cb200_gather_close": (C.c_int, [C.c_void_p]),
    "cb200_gather_push": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_gather_flush": (C.c_int, [C.c_void_p, C.c_int]),
    "cb200_host_alloc": (C.c_void_p, [C.c_size_t]),
    "cb200_host_alloc_batch": (C.c_void_p, [C.c_size_t, C.c_size_t]),
    "cb200_host_free": (None, [C.c_void_p]),
    "cb200_launch_count": (C.c_uint64, []),
    "cb200_profile_enable": (C.c_int, [C.c_int]),
    "cb200_profile_kernel_count": (C.c_int, []),
    "cb200_profile_kernel_name": (C.c_char_p, [C.c_int]),
    "cb200_profile_read": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int]),
    "cb200_kyber_ntt": (C.c_int, [C.c_void_p, C.c_size_t, C.c_int]),
    "cb200_kyber_mulhat": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_kyber_dot": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_size_t]),
    "cb200_kyber_poly_op": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_dil_ntt": (C.c_int, [C.c_void_p, C.c_size_t, C.c_int]),
    "cb200_dil_mulhat": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_dil_dot": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_size_t]),
    "cb200_dil_poly_op": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_dil_exceeds": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t]),
    "cb200_keccak_f1600": (C.c_int, [C.c_void_p, C.c_size_t, C.c_int]),
    "cb200_sha3": (C.c_int, [C.c_int, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t]),
    "cb200_kyber_derive_uniform": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]),
    "cb200_kyber_derive_noise": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]),
    "cb200_kyber_pack": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_kyber_unpack": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_kyber_compress": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_size_t]),
    "cb200_kyber_decompress": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_size_t]),
    "cb200_dil_derive_uniform": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]),
    "cb200_dil_derive_leq_eta": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]),
    "cb200_dil_derive_le_gamma1": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]),
    "cb200_dil_derive_ball": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t]),
    "cb200_dil_power2round": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_dil_pack_le16": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_mlkem_encaps": (C.c_int, [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_size_t]),
    "cb200_mlkem_encaps_push": (C.c_int, [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    "cb200_kyber_kem_keygen": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_kyber_kem_encaps": (C.c_int, [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_kyber_kem_decaps": (C.c_int, [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_x25519": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_x448": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_xwing_keygen": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_xwing_encaps": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_xwing_decaps": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_hybrid_keygen": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_hybrid_encaps": (C.c_int, [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_hybrid_decaps": (C.c_int, [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_hybrid_public_key_size": (C.c_size_t, [C.c_int]),
    "cb200_hybrid_private_key_size": (C.c_size_t, [C.c_int]),
    "cb200_hybrid_ciphertext_size": (C.c_size_t, [C.c_int]),
    "cb200_hybrid_shared_key_size": (C.c_size_t, [C.c_int]),
    "cb200_hybrid_seed_size": (C.c_size_t, [C.c_int]),
    "cb200_hybrid_encapsulation_seed_size": (C.c_size_t, [C.c_int]),
    "cb200_hpke_keygen": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_hpke_encaps": (C.c_int, [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_size_t]),
    "cb200_hpke_decaps": (C.c_int, [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_hpke_auth_encaps": (C.c_int, [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_hpke_auth_decaps": (C.c_int, [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p,
                                         C.c_void_p, C.c_size_t]),
    "cb200_hpke_public_key_size": (C.c_size_t, [C.c_int]),
    "cb200_hpke_private_key_size": (C.c_size_t, [C.c_int]),
    "cb200_hpke_ciphertext_size": (C.c_size_t, [C.c_int]),
    "cb200_hpke_shared_key_size": (C.c_size_t, [C.c_int]),
    "cb200_hpke_seed_size": (C.c_size_t, [C.c_int]),
    "cb200_hpke_encapsulation_seed_size": (C.c_size_t, [C.c_int]),
    "cb200_p256": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_hpke_p256_keygen": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_hpke_p256_encaps": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_size_t]),
    "cb200_hpke_p256_decaps": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_hpke_p256_auth_encaps": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_hpke_p256_auth_decaps": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p,
                                              C.c_void_p, C.c_size_t]),
    "cb200_hpke_p256_public_key_size": (C.c_size_t, []),
    "cb200_hpke_p256_private_key_size": (C.c_size_t, []),
    "cb200_hpke_p256_ciphertext_size": (C.c_size_t, []),
    "cb200_hpke_p256_shared_key_size": (C.c_size_t, []),
    "cb200_hpke_p256_seed_size": (C.c_size_t, []),
    "cb200_hpke_p256_encapsulation_seed_size": (C.c_size_t, []),
    "cb200_p384": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_oprf_element_size": (C.c_size_t, [C.c_int]),
    "cb200_oprf_scalar_size": (C.c_size_t, [C.c_int]),
    "cb200_oprf_output_size": (C.c_size_t, [C.c_int]),
    "cb200_oprf_proof_size": (C.c_size_t, [C.c_int]),
    "cb200_oprf_derive_key": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                        C.c_size_t]),
    "cb200_oprf_evaluate": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p,
                                      C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_oprf_full_evaluate": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_brsa_modulus_bytes": (C.c_size_t, [C.c_char_p, C.c_size_t]),
    "cb200_brsa_blind_sign": (C.c_int, [C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t,
                                        C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t,
                                        C.c_char_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_brsa_verify": (C.c_int, [C.c_int, C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_hpke_p384_keygen": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_hpke_p384_encaps": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_size_t]),
    "cb200_hpke_p384_decaps": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_hpke_p384_auth_encaps": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_hpke_p384_auth_decaps": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p,
                                              C.c_void_p, C.c_size_t]),
    "cb200_hpke_p384_public_key_size": (C.c_size_t, []),
    "cb200_hpke_p384_private_key_size": (C.c_size_t, []),
    "cb200_hpke_p384_ciphertext_size": (C.c_size_t, []),
    "cb200_hpke_p384_shared_key_size": (C.c_size_t, []),
    "cb200_hpke_p384_seed_size": (C.c_size_t, []),
    "cb200_hpke_p384_encapsulation_seed_size": (C.c_size_t, []),
    "cb200_p521": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_hpke_p521_keygen": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_hpke_p521_encaps": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_size_t]),
    "cb200_hpke_p521_decaps": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_hpke_p521_auth_encaps": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_hpke_p521_auth_decaps": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p,
                                              C.c_void_p, C.c_size_t]),
    "cb200_hpke_p521_public_key_size": (C.c_size_t, []),
    "cb200_hpke_p521_private_key_size": (C.c_size_t, []),
    "cb200_hpke_p521_ciphertext_size": (C.c_size_t, []),
    "cb200_hpke_p521_shared_key_size": (C.c_size_t, []),
    "cb200_hpke_p521_seed_size": (C.c_size_t, []),
    "cb200_hpke_p521_encapsulation_seed_size": (C.c_size_t, []),
    "cb200_frodo640shake_keygen": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_frodo640shake_encaps": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_frodo640shake_decaps": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_frodo640shake_public_key_size": (C.c_size_t, []),
    "cb200_frodo640shake_private_key_size": (C.c_size_t, []),
    "cb200_frodo640shake_ciphertext_size": (C.c_size_t, []),
    "cb200_frodo640shake_shared_key_size": (C.c_size_t, []),
    "cb200_frodo640shake_seed_size": (C.c_size_t, []),
    "cb200_frodo640shake_encapsulation_seed_size": (C.c_size_t, []),
    "cb200_mldsa_sign": (C.c_int, [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p]),
    "cb200_mldsa_verify": (C.c_int, [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                     C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]),
    "cb200_mldsa_keygen": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_mldsa_public_key_size": (C.c_size_t, [C.c_int]),
    "cb200_mldsa_private_key_size": (C.c_size_t, [C.c_int]),
    "cb200_mldsa_signature_size": (C.c_size_t, [C.c_int]),
    "cb200_mldsa65_sign": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p]),
    "cb200_mldsa65_verify": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p,
                                       C.c_void_p, C.c_size_t, C.c_int]),
    "cb200_mldsa65_keygen": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_mldsa65_public_key_size": (C.c_size_t, []),
    "cb200_mldsa65_signature_size": (C.c_size_t, []),
    "cb200_mldsa65_private_key_size": (C.c_size_t, []),
    "cb200_ed25519_keygen": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_ed25519_sign": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_ed25519_verify": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_ed25519_public_key_size": (C.c_size_t, []),
    "cb200_ed25519_private_key_size": (C.c_size_t, []),
    "cb200_ed25519_signature_size": (C.c_size_t, []),
    "cb200_ed25519_seed_size": (C.c_size_t, []),
    "cb200_eddilithium2_keygen": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_eddilithium2_sign": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_size_t]),
    "cb200_eddilithium2_verify": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_size_t]),
    "cb200_eddilithium2_public_key_size": (C.c_size_t, []),
    "cb200_eddilithium2_private_key_size": (C.c_size_t, []),
    "cb200_eddilithium2_signature_size": (C.c_size_t, []),
    "cb200_eddilithium2_seed_size": (C.c_size_t, []),
    "cb200_ed448_keygen": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_ed448_sign": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p,
                                   C.c_size_t]),
    "cb200_ed448_verify": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p,
                                     C.c_void_p, C.c_size_t]),
    "cb200_ed448_public_key_size": (C.c_size_t, []),
    "cb200_ed448_private_key_size": (C.c_size_t, []),
    "cb200_ed448_signature_size": (C.c_size_t, []),
    "cb200_ed448_seed_size": (C.c_size_t, []),
    "cb200_eddilithium3_keygen": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_eddilithium3_sign": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_size_t]),
    "cb200_eddilithium3_verify": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_size_t]),
    "cb200_eddilithium3_public_key_size": (C.c_size_t, []),
    "cb200_eddilithium3_private_key_size": (C.c_size_t, []),
    "cb200_eddilithium3_signature_size": (C.c_size_t, []),
    "cb200_eddilithium3_seed_size": (C.c_size_t, []),
    "cb200_mlkem_decaps": (C.c_int, [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_mlkem_keygen": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cb200_mlkem_private_key_size": (C.c_size_t, [C.c_int]),
    "cb200_mlkem_public_key_size": (C.c_size_t, [C.c_int]),
    "cb200_mlkem_ciphertext_size": (C.c_size_t, [C.c_int]),
}

_lib = None


class Cb200Error(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"cb200 error {code}: {msg}")
        self.code = code


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            # Not a fallback: the only way forward is the CUDA library itself, so build it (nvcc, sm_90a).
            try:
                from .build import build_library
                build_library()
            except Exception as e:  # pragma: no cover
                raise ImportError(
                    f"{LIB_PATH} is missing and could not be built with nvcc ({e}). "
                    "circl_b200 has no CPU fallback.") from e
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            if not hasattr(L, name):
                continue  # test_abi reports missing symbols
            f = getattr(L, name)
            f.restype = res
            f.argtypes = args
        _lib = L
    return _lib


def check(rc: int) -> None:
    if rc != 0:
        raise Cb200Error(rc, lib().cb200_last_error().decode())
