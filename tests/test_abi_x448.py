"""CPU-only: the X448 entry points and the X448 hybrid schemes fail loudly without a device, and their sizes."""
import numpy as np
import pytest


def test_x448_entry_points_fail_without_a_device():
    from circl_b200 import _ffi, x448
    if _ffi.lib().cb200_device_count() > 0:
        pytest.skip("a CUDA device is visible")
    k = np.zeros((2, 56), dtype=np.uint8)
    for call in (lambda: x448.x448_keygen(k),
                 lambda: x448.x448_shared(k, k),
                 lambda: x448.ByName("Kyber768-X448").DeriveKeyPairBatch(np.zeros((2, 64), dtype=np.uint8)),
                 lambda: x448.ByName("Kyber1024-X448").DeriveKeyPairBatch(np.zeros((2, 64), dtype=np.uint8))):
        with pytest.raises(_ffi.Cb200Error) as ei:
            call()
        assert "not initialised" in str(ei.value)


def test_hybrid_size_getters():
    from circl_b200._ffi import lib
    L = lib()
    sizes = {i: (L.cb200_hybrid_public_key_size(i), L.cb200_hybrid_private_key_size(i), L.cb200_hybrid_ciphertext_size(i),
                 L.cb200_hybrid_shared_key_size(i), L.cb200_hybrid_seed_size(i), L.cb200_hybrid_encapsulation_seed_size(i))
             for i in range(6)}
    assert sizes[0] == (1216, 2432, 1120, 64, 64, 32)
    assert sizes[1] == (1216, 2432, 1120, 64, 64, 32)
    assert sizes[2] == (832, 1664, 800, 64, 64, 32)
    assert sizes[3] == (1240, 2456, 1144, 88, 64, 56)
    assert sizes[4] == (1624, 3224, 1624, 88, 64, 56)
    assert sizes[5] == (0, 0, 0, 0, 0, 0)


def test_registry_names_match_the_reference():
    # kem/schemes/schemes.go:48-54, kem/hybrid/hybrid.go:83-93
    from circl_b200 import hybrid, x448
    assert [s.Name() for s in x448.All()] == ["Kyber768-X448", "Kyber1024-X448"]
    assert x448.ByName("kyber1024-x448") is x448.All()[1] and x448.ByName("Kyber768-X25519") is None
    assert all(isinstance(s, hybrid.Hybrid) for s in x448.All())
    s = x448.ByName("Kyber768-X448")
    assert (s.SeedSize(), s.EncapsulationSeedSize(), s.SharedKeySize()) == (64, 56, 88)
