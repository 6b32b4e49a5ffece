"""CPU-only: the FrodoKEM-640-SHAKE entry points are exported and fail loudly without a device, the six sizes, the
registry, and the errors that hold before any device work.  The existing registries are unchanged."""
import ctypes as C

import numpy as np
import pytest

ENTRY = ["cb200_frodo640shake_keygen", "cb200_frodo640shake_encaps", "cb200_frodo640shake_decaps"]
SIZES = ["public_key", "private_key", "ciphertext", "shared_key", "seed", "encapsulation_seed"]


def test_exports_and_sizes():
    from circl_b200._ffi import lib
    L = C.CDLL(lib()._name)
    for name in ENTRY + [f"cb200_frodo640shake_{s}_size" for s in SIZES]:
        assert hasattr(L, name), name
    # frodo.go:32-51
    assert tuple(getattr(lib(), f"cb200_frodo640shake_{s}_size")() for s in SIZES) == (9616, 19888, 9720, 16, 48, 16)


def test_entry_points_fail_without_a_device():
    from circl_b200 import _ffi, frodo
    if _ffi.lib().cb200_device_count() > 0:
        pytest.skip("a CUDA device is visible")
    s = frodo.Scheme()
    for call in (lambda: s.DeriveKeyPairBatch(np.zeros((2, 48), np.uint8)),
                 lambda: s.EncapsulateBatch(np.zeros((2, 9616), np.uint8), np.zeros((2, 16), np.uint8)),
                 lambda: s.DecapsulateBatch(np.zeros((2, 19888), np.uint8), np.zeros((2, 9720), np.uint8))):
        with pytest.raises(_ffi.Cb200Error) as ei:
            call()
        assert ei.value.code == -2 and "not initialised" in str(ei.value)


def test_registry():
    from circl_b200 import frodo, hpke, hybrid, mlkem, x448
    assert [s.Name() for s in frodo.All()] == ["FrodoKEM-640-SHAKE"]
    assert frodo.ByName("frodokem-640-shake") is frodo.Scheme() is frodo.All()[0]
    assert frodo.ByName("FrodoKEM-640-AES") is None and frodo.ByName("X-Wing") is None
    assert [s.Name() for s in hybrid.All()] == ["X-Wing", "X25519MLKEM768", "Kyber768-X25519", "Kyber512-X25519"]
    assert [s.Name() for s in x448.All()] == ["Kyber768-X448", "Kyber1024-X448"]
    assert [s.Name() for s in hpke.All()] == ["HPKE_KEM_X25519_HKDF_SHA256", "HPKE_KEM_X448_HKDF_SHA512"]
    assert "FrodoKEM-640-SHAKE" not in [s.Name() for s in mlkem.All()]
    for m in (hybrid, x448, hpke, mlkem):
        assert m.ByName("FrodoKEM-640-SHAKE") is None


def test_errors_before_any_device_work():
    from circl_b200 import frodo, hpke, mlkem
    s = frodo.Scheme()
    other = hpke.All()[0]
    pk, sk = s.UnmarshalBinaryPublicKey(bytes(9616)), s.UnmarshalBinaryPrivateKey(bytes(19888))
    assert sk.Public().MarshalBinary() == bytes(9616) and sk.Public().Equal(pk)
    with pytest.raises(mlkem.ErrPubKeySize):
        s.UnmarshalBinaryPublicKey(bytes(9615))
    with pytest.raises(mlkem.ErrPrivKeySize):
        s.UnmarshalBinaryPrivateKey(bytes(19889))
    with pytest.raises(mlkem.ErrSeedSize):
        s.DeriveKeyPair(bytes(32))
    with pytest.raises(mlkem.ErrSeedSize):
        s.EncapsulateDeterministically(pk, bytes(32))
    with pytest.raises(mlkem.ErrCiphertextSize):
        s.Decapsulate(sk, bytes(9719))
    with pytest.raises(mlkem.ErrTypeMismatch):
        s.Decapsulate(other.UnmarshalBinaryPrivateKey(bytes(32)), bytes(9720))
    with pytest.raises(mlkem.ErrTypeMismatch):
        s.EncapsulateDeterministically(other.UnmarshalBinaryPublicKey(bytes(32)), bytes(16))
    # the reference's order: the seed or ciphertext length before the key's type
    with pytest.raises(mlkem.ErrCiphertextSize):
        s.Decapsulate(other.UnmarshalBinaryPrivateKey(bytes(32)), bytes(1))
    with pytest.raises(mlkem.ErrSeedSize):
        s.EncapsulateDeterministically(other.UnmarshalBinaryPublicKey(bytes(32)), bytes(1))
    with pytest.raises(mlkem.ErrPrivKeySize):
        s.DecapsulateBatch(np.zeros((2, 100), np.uint8), np.zeros((2, 9720), np.uint8))
