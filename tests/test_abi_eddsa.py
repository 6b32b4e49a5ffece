"""CPU-only: the Ed25519 and Ed25519-Dilithium2 entry points fail loudly without a device, their sizes, and the
registry names and order."""
import numpy as np
import pytest


def test_entry_points_fail_without_a_device():
    from circl_b200 import _ffi, eddsa
    if _ffi.lib().cb200_device_count() > 0:
        pytest.skip("a CUDA device is visible")
    seeds = np.zeros((2, 32), dtype=np.uint8)
    ed, edd = eddsa.ByName("Ed25519"), eddsa.ByName("Ed25519-Dilithium2")
    for call in (lambda: ed.DeriveKeyBatch(seeds),
                 lambda: ed.SignBatch(np.zeros((2, 64), dtype=np.uint8), [b"a", b"b"]),
                 lambda: ed.VerifyBatch(np.zeros((2, 32), dtype=np.uint8), [b"a", b"b"], np.zeros((2, 64), dtype=np.uint8)),
                 lambda: edd.DeriveKeyBatch(seeds),
                 lambda: edd.SignBatch(np.zeros((2, 2560), dtype=np.uint8), [b"a", b"b"]),
                 lambda: edd.VerifyBatch(np.zeros((2, 1344), dtype=np.uint8), [b"a", b"b"],
                                         np.zeros((2, 2484), dtype=np.uint8))):
        with pytest.raises(_ffi.Cb200Error) as ei:
            call()
        assert ei.value.code == -2 and "not initialised" in str(ei.value)


def test_sizes():
    from circl_b200._ffi import lib
    L = lib()
    assert (L.cb200_ed25519_public_key_size(), L.cb200_ed25519_private_key_size(), L.cb200_ed25519_signature_size(),
            L.cb200_ed25519_seed_size()) == (32, 64, 64, 32)
    # eddilithium.go:16-28: mode2 sizes plus the Ed25519 public key, seed and signature
    assert (L.cb200_eddilithium2_public_key_size(), L.cb200_eddilithium2_private_key_size(),
            L.cb200_eddilithium2_signature_size(), L.cb200_eddilithium2_seed_size()) == (1312 + 32, 2528 + 32, 2420 + 64, 32)


def test_registry_names_and_order():
    # sign/schemes/schemes.go:31-35 lists Ed25519 and Ed25519-Dilithium2 first; mldsa keeps its own list
    from circl_b200 import eddsa, mldsa
    assert [s.Name() for s in eddsa.All()] == ["Ed25519", "Ed25519-Dilithium2"]
    assert eddsa.ByName("ed25519") is eddsa.All()[0] and eddsa.ByName("Ed448") is None
    assert [s.Name() for s in mldsa.All()] == ["ML-DSA-44", "ML-DSA-65", "ML-DSA-87", "Dilithium2", "Dilithium3", "Dilithium5"]
    for s in eddsa.All():
        assert not s.SupportsContext()
    with pytest.raises(eddsa.ErrContextNotSupported):
        eddsa.ByName("Ed25519").SignBatch(np.zeros((1, 64), dtype=np.uint8), [b"m"], ctx=b"c")
    assert eddsa.ByName("Ed25519").Verify(eddsa.ByName("Ed25519").UnmarshalBinaryPublicKey(bytes(32)), b"m", bytes(63)) is False
