"""CPU-only: the HPKE DHKEM entry points are exported and fail loudly without a device, their sizes per id (0 for an
unknown id), the registry names and order, and the errors that hold before any device work.  The existing registries
are unchanged."""
import ctypes as C

import numpy as np
import pytest

ENTRY = ["cb200_hpke_keygen", "cb200_hpke_encaps", "cb200_hpke_decaps", "cb200_hpke_auth_encaps", "cb200_hpke_auth_decaps"]
SIZES = ["public_key", "private_key", "ciphertext", "shared_key", "seed", "encapsulation_seed"]


def test_exports_and_sizes():
    from circl_b200._ffi import lib
    L = C.CDLL(lib()._name)
    for name in ENTRY + [f"cb200_hpke_{s}_size" for s in SIZES]:
        assert hasattr(L, name), name
    L = lib()
    # xkem.go:20-24 and kembase.go:34: X25519 everything 32; X448 everything 56 except the 64-byte SHA-512 secret
    want = {0x20: (32, 32, 32, 32, 32, 32), 0x21: (56, 56, 56, 64, 56, 56)}
    for kid, sizes in want.items():
        assert tuple(getattr(L, f"cb200_hpke_{s}_size")(kid) for s in SIZES) == sizes
    for bad in (0, 0x10, 0x11, 0x12, 0x22, 0x30, -1):
        assert all(getattr(L, f"cb200_hpke_{s}_size")(bad) == 0 for s in SIZES)


def test_entry_points_fail_without_a_device():
    from circl_b200 import _ffi, hpke
    if _ffi.lib().cb200_device_count() > 0:
        pytest.skip("a CUDA device is visible")
    for s in hpke.All():
        n = s.SeedSize()
        z = np.zeros((2, n), dtype=np.uint8)
        for call in (lambda: s.DeriveKeyPairBatch(z), lambda: s.EncapsulateBatch(z, z), lambda: s.DecapsulateBatch(z, z),
                     lambda: s.AuthEncapsulateBatch(z, z, z), lambda: s.AuthDecapsulateBatch(z, z, z)):
            with pytest.raises(_ffi.Cb200Error) as ei:
                call()
            assert ei.value.code == -2 and "not initialised" in str(ei.value)


def test_registry_names_and_order():
    from circl_b200 import hpke, hybrid, x448
    assert [s.Name() for s in hpke.All()] == ["HPKE_KEM_X25519_HKDF_SHA256", "HPKE_KEM_X448_HKDF_SHA512"]
    assert hpke.ByName("hpke_kem_x25519_hkdf_sha256") is hpke.All()[0]
    assert hpke.ByName("HPKE_KEM_X448_HKDF_SHA512") is hpke.All()[1]
    assert hpke.ByName("HPKE_KEM_P256_HKDF_SHA256") is None and hpke.ByName("X-Wing") is None
    assert [s.Name() for s in hybrid.All()] == ["X-Wing", "X25519MLKEM768", "Kyber768-X25519", "Kyber512-X25519"]
    assert [s.Name() for s in x448.All()] == ["Kyber768-X448", "Kyber1024-X448"]
    assert hybrid.ByName("HPKE_KEM_X25519_HKDF_SHA256") is None and x448.ByName("HPKE_KEM_X448_HKDF_SHA512") is None


def test_errors_before_any_device_work():
    from circl_b200 import hpke, mlkem
    a, b = hpke.All()
    # Decapsulate parses ct as a public key: kem.ErrPubKeySize, not ErrCiphertextSize (kembase.go:222)
    sk = a.UnmarshalBinaryPrivateKey(bytes(32))
    with pytest.raises(mlkem.ErrPubKeySize):
        a.Decapsulate(sk, bytes(31))
    with pytest.raises(mlkem.ErrPubKeySize):
        a.AuthDecapsulate(sk, bytes(33), a.UnmarshalBinaryPublicKey(bytes(32)))
    with pytest.raises(mlkem.ErrSeedSize):
        b.DeriveKeyPair(bytes(32))
    with pytest.raises(mlkem.ErrSeedSize):
        a.EncapsulateDeterministically(a.UnmarshalBinaryPublicKey(bytes(32)), bytes(56))
    # UnmarshalBinary* check the length only
    assert b.UnmarshalBinaryPublicKey(bytes(56)).MarshalBinary() == bytes(56)
    with pytest.raises(mlkem.ErrPubKeySize):
        b.UnmarshalBinaryPublicKey(bytes(57))
    with pytest.raises(mlkem.ErrPrivKeySize):
        a.UnmarshalBinaryPrivateKey(bytes(56))
    with pytest.raises(mlkem.ErrTypeMismatch):
        a.Decapsulate(b.UnmarshalBinaryPrivateKey(bytes(56)), bytes(32))
    # the reference's order: the encapsulation (parsed as a public key) or the seed before the key's type
    with pytest.raises(mlkem.ErrPubKeySize):
        a.Decapsulate(b.UnmarshalBinaryPrivateKey(bytes(56)), bytes(31))
    with pytest.raises(mlkem.ErrPubKeySize):
        a.AuthDecapsulate(b.UnmarshalBinaryPrivateKey(bytes(56)), bytes(31), b.UnmarshalBinaryPublicKey(bytes(56)))
    with pytest.raises(mlkem.ErrSeedSize):
        a.EncapsulateDeterministically(b.UnmarshalBinaryPublicKey(bytes(56)), bytes(31))
    with pytest.raises(mlkem.ErrSeedSize):
        a.AuthEncapsulateDeterministically(b.UnmarshalBinaryPublicKey(bytes(56)), b.UnmarshalBinaryPrivateKey(bytes(56)),
                                           bytes(31))
    assert (a.SharedKeySize(), b.SharedKeySize()) == (32, 64)
    assert issubclass(hpke.ErrInvalidKEMSharedSecret, mlkem.KemError)
