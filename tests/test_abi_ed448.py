"""CPU-only: the Ed448 and Ed448-Dilithium3 entry points fail loudly without a device, their sizes, the registry names
and order, and the context rules that hold before any device work."""
import numpy as np
import pytest


def test_entry_points_fail_without_a_device():
    from circl_b200 import _ffi, ed448
    if _ffi.lib().cb200_device_count() > 0:
        pytest.skip("a CUDA device is visible")
    seeds = np.zeros((2, 57), dtype=np.uint8)
    ed, edd = ed448.ByName("Ed448"), ed448.ByName("Ed448-Dilithium3")
    for call in (lambda: ed.DeriveKeyBatch(seeds),
                 lambda: ed.SignBatch(np.zeros((2, 114), dtype=np.uint8), [b"a", b"b"], ctx=b"c"),
                 lambda: ed.VerifyBatch(np.zeros((2, 57), dtype=np.uint8), [b"a", b"b"], np.zeros((2, 114), dtype=np.uint8)),
                 lambda: edd.DeriveKeyBatch(seeds),
                 lambda: edd.SignBatch(np.zeros((2, 4057), dtype=np.uint8), [b"a", b"b"]),
                 lambda: edd.VerifyBatch(np.zeros((2, 2009), dtype=np.uint8), [b"a", b"b"],
                                         np.zeros((2, 3407), dtype=np.uint8))):
        with pytest.raises(_ffi.Cb200Error) as ei:
            call()
        assert ei.value.code == -2 and "not initialised" in str(ei.value)


def test_sizes():
    from circl_b200._ffi import lib
    L = lib()
    # ed448.go:41-52
    assert (L.cb200_ed448_public_key_size(), L.cb200_ed448_private_key_size(), L.cb200_ed448_signature_size(),
            L.cb200_ed448_seed_size()) == (57, 114, 114, 57)
    # eddilithium.go:16-28: mode3 sizes plus the Ed448 public key, seed and signature
    assert (L.cb200_eddilithium3_public_key_size(), L.cb200_eddilithium3_private_key_size(),
            L.cb200_eddilithium3_signature_size(), L.cb200_eddilithium3_seed_size()) == (1952 + 57, 4000 + 57, 3293 + 114, 57)


def test_registry_names_and_order():
    # sign/schemes/schemes.go:31-54 lists Ed448 second and Ed448-Dilithium3 fourth; eddsa and mldsa keep their lists
    from circl_b200 import ed448, eddsa, mldsa
    assert [s.Name() for s in ed448.All()] == ["Ed448", "Ed448-Dilithium3"]
    assert ed448.ByName("ED448") is ed448.All()[0] and ed448.ByName("ed448-DILITHIUM3") is ed448.All()[1]
    assert ed448.ByName("Ed25519") is None
    assert [s.Name() for s in eddsa.All()] == ["Ed25519", "Ed25519-Dilithium2"] and eddsa.ByName("Ed448") is None
    assert [s.Name() for s in mldsa.All()] == ["ML-DSA-44", "ML-DSA-65", "ML-DSA-87", "Dilithium2", "Dilithium3", "Dilithium5"]
    ed, edd = ed448.All()
    assert ed.SupportsContext() and not edd.SupportsContext()
    assert (ed.PublicKeySize(), ed.PrivateKeySize(), ed.SignatureSize(), ed.SeedSize()) == (57, 114, 114, 57)


def test_context_errors_before_any_device_work():
    from circl_b200 import ed448
    ed, edd = ed448.All()
    with pytest.raises(ed448.ErrContextTooLong):
        ed.SignBatch(np.zeros((1, 114), dtype=np.uint8), [b"m"], ctx=bytes(256))
    with pytest.raises(ed448.ErrContextNotSupported):
        edd.SignBatch(np.zeros((1, 4057), dtype=np.uint8), [b"m"], ctx=b"c")
    with pytest.raises(ed448.ErrContextNotSupported):
        edd.Verify(edd.UnmarshalBinaryPublicKey(bytes(2009)), b"m", bytes(3407), ed448.SignatureOpts(b"c"))
    assert ed.Verify(ed.UnmarshalBinaryPublicKey(bytes(57)), b"m", bytes(113)) is False
    with pytest.raises(ed448.ErrPubKeySize):
        ed.UnmarshalBinaryPublicKey(bytes(56))
    with pytest.raises(ed448.ErrPrivKeySize):
        edd.SignBatch(ed.UnmarshalBinaryPrivateKey(bytes(114)), [b"m"])  # a key of the other scheme
