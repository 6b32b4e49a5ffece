"""CPU-only: the P-256 entry points are exported and fail loudly without a device, their sizes, the registry, the
host-side key validation and the errors that hold before any device work.  0x10 stays unknown to the generic HPKE
entry points and registries."""
import ctypes as C

import numpy as np
import pytest

ENTRY = ["cb200_p256", "cb200_hpke_p256_keygen", "cb200_hpke_p256_encaps", "cb200_hpke_p256_decaps",
         "cb200_hpke_p256_auth_encaps", "cb200_hpke_p256_auth_decaps"]
SIZES = ["public_key", "private_key", "ciphertext", "shared_key", "seed", "encapsulation_seed"]
N = 0xffffffff00000000ffffffffffffffffbce6faada7179e84f3b9cac2fc632551
G = bytes.fromhex("046b17d1f2e12c4247f8bce6e563a440f277037d812deb33a0f4a13945d898c296"
                  "4fe342e2fe1a7f9b8ee7eb4a7c0f9e162bce33576b315ececbb6406837bf51f5")


def test_exports_and_sizes():
    from circl_b200._ffi import lib
    L = C.CDLL(lib()._name)
    for name in ENTRY + [f"cb200_hpke_p256_{s}_size" for s in SIZES]:
        assert hasattr(L, name), name
    L = lib()
    assert [getattr(L, f"cb200_hpke_p256_{s}_size")() for s in SIZES] == [65, 32, 65, 32, 32, 32]
    assert all(getattr(L, f"cb200_hpke_{s}_size")(0x10) == 0 for s in SIZES)


def test_registry():
    from circl_b200 import hpke, p256
    assert [s.Name() for s in p256.All()] == ["HPKE_KEM_P256_HKDF_SHA256"]
    assert p256.ByName("hpke_kem_p256_hkdf_sha256") is p256.All()[0]
    assert p256.ByName("HPKE_KEM_X25519_HKDF_SHA256") is None
    assert hpke.ByName("HPKE_KEM_P256_HKDF_SHA256") is None and len(hpke.All()) == 2
    s = p256.All()[0]
    assert isinstance(s, hpke.DHKEM)
    assert (s.PublicKeySize(), s.PrivateKeySize(), s.CiphertextSize(), s.SharedKeySize(), s.SeedSize(),
            s.EncapsulationSeedSize()) == (65, 32, 65, 32, 32, 32)


def test_entry_points_fail_without_a_device():
    from circl_b200 import _ffi, p256
    if _ffi.lib().cb200_device_count() > 0:
        pytest.skip("a CUDA device is visible")
    s = p256.All()[0]
    z32, z65 = np.zeros((2, 32), dtype=np.uint8), np.zeros((2, 65), dtype=np.uint8)
    for call in (lambda: s.DeriveKeyPairBatch(z32), lambda: s.EncapsulateBatch(z65, z32), lambda: s.DecapsulateBatch(z32, z65),
                 lambda: s.AuthEncapsulateBatch(z65, z32, z32), lambda: s.AuthDecapsulateBatch(z32, z65, z65),
                 lambda: p256.p256_keygen(z32), lambda: p256.p256_shared(z32, z65)):
        with pytest.raises(_ffi.Cb200Error) as ei:
            call()
        assert ei.value.code == -2 and "not initialised" in str(ei.value)


def test_unmarshal_validates_like_crypto_ecdh():
    from circl_b200 import mlkem, p256
    s = p256.All()[0]
    assert issubclass(p256.ErrInvalidKEMPublicKey, mlkem.KemError)
    assert issubclass(p256.ErrInvalidKEMPrivateKey, mlkem.KemError)
    assert s.UnmarshalBinaryPublicKey(G).MarshalBinary() == G
    for bad in (b"\x02" + G[1:], bytes(65), G[:64] + bytes([G[64] ^ 1])):
        with pytest.raises(p256.ErrInvalidKEMPublicKey):
            s.UnmarshalBinaryPublicKey(bad)
    with pytest.raises(mlkem.ErrPubKeySize):
        s.UnmarshalBinaryPublicKey(G[:33])
    assert s.UnmarshalBinaryPrivateKey((N - 1).to_bytes(32, "big")).MarshalBinary() == (N - 1).to_bytes(32, "big")
    for bad in (0, N, 2**256 - 1):
        with pytest.raises(p256.ErrInvalidKEMPrivateKey):
            s.UnmarshalBinaryPrivateKey(bad.to_bytes(32, "big"))
    with pytest.raises(mlkem.ErrPrivKeySize):
        s.UnmarshalBinaryPrivateKey(bytes(65))


def test_errors_before_any_device_work():
    from circl_b200 import hpke, mlkem, p256
    s, x = p256.All()[0], hpke.All()[0]
    sk = s.UnmarshalBinaryPrivateKey((7).to_bytes(32, "big"))
    pk = s.UnmarshalBinaryPublicKey(G)
    # Decap parses enc as a public key first (kembase.go:222): the size, then the point
    with pytest.raises(mlkem.ErrPubKeySize):
        s.Decapsulate(sk, bytes(32))
    with pytest.raises(p256.ErrInvalidKEMPublicKey):
        s.Decapsulate(sk, bytes(65))
    with pytest.raises(mlkem.ErrSeedSize):
        s.DeriveKeyPair(bytes(65))
    with pytest.raises(mlkem.ErrSeedSize):
        s.EncapsulateDeterministically(pk, bytes(31))
    with pytest.raises(mlkem.ErrTypeMismatch):
        s.Decapsulate(x.UnmarshalBinaryPrivateKey(bytes(32)), G)
    with pytest.raises(mlkem.ErrTypeMismatch):
        s.AuthEncapsulateDeterministically(pk, x.UnmarshalBinaryPrivateKey(bytes(32)), bytes(32))
