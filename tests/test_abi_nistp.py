"""CPU-only: the P-384 and P-521 entry points are exported and fail loudly without a device, their sizes, the
registries, the host-side key validation and the errors that hold before any device work.  0x11 and 0x12 stay unknown
to the generic HPKE entry points and registries, and hpke.All() / p256.All() are unchanged."""
import ctypes as C
import importlib

import numpy as np
import pytest

from nistp_model import CURVES, enc

SIZES = ["public_key", "private_key", "ciphertext", "shared_key", "seed", "encapsulation_seed"]
WANT = {384: [97, 48, 97, 48, 48, 48], 521: [133, 66, 133, 64, 66, 66]}
NAMES = {384: "HPKE_KEM_P384_HKDF_SHA384", 521: "HPKE_KEM_P521_HKDF_SHA512"}


@pytest.mark.parametrize("bits", [384, 521])
def test_exports_and_sizes(bits):
    from circl_b200._ffi import lib
    L = C.CDLL(lib()._name)
    pre = f"cb200_hpke_p{bits}_"
    for name in [f"cb200_p{bits}"] + [pre + e for e in ("keygen", "encaps", "decaps", "auth_encaps", "auth_decaps")]:
        assert hasattr(L, name), name
    L = lib()
    assert [getattr(L, f"{pre}{s}_size")() for s in SIZES] == WANT[bits]
    assert all(getattr(L, f"cb200_hpke_{s}_size")(CURVES[bits].kem_id) == 0 for s in SIZES)


def test_generic_entry_points_reject_the_ids():
    from circl_b200 import _ffi
    L = _ffi.lib()
    z = np.zeros(256, np.uint8)
    p = z.ctypes.data
    for ident in (0x11, 0x12):
        assert L.cb200_hpke_keygen(ident, p, p, p, 1) != 0


def test_registries():
    from circl_b200 import hpke, p256, p384, p521
    assert [s.Name() for s in p384.All()] == [NAMES[384]] and [s.Name() for s in p521.All()] == [NAMES[521]]
    assert p384.ByName(NAMES[384].lower()) is p384.All()[0] and p521.ByName(NAMES[521].lower()) is p521.All()[0]
    assert p384.ByName(NAMES[521]) is None and p521.ByName("HPKE_KEM_P256_HKDF_SHA256") is None
    assert len(hpke.All()) == 2 and all(hpke.ByName(n) is None for n in NAMES.values())
    assert [s.Name() for s in p256.All()] == ["HPKE_KEM_P256_HKDF_SHA256"]
    assert isinstance(p256.All()[0], p256.P256DHKEM)
    assert not isinstance(p384.All()[0], p256.P256DHKEM) and not isinstance(p521.All()[0], p256.P256DHKEM)
    assert p384.ErrInvalidKEMPublicKey is p256.ErrInvalidKEMPublicKey
    assert p521.ErrInvalidKEMPrivateKey is p256.ErrInvalidKEMPrivateKey
    for bits, m in ((384, p384), (521, p521)):
        s = m.All()[0]
        assert isinstance(s, hpke.DHKEM)
        assert [s.PublicKeySize(), s.PrivateKeySize(), s.CiphertextSize(), s.SharedKeySize(), s.SeedSize(),
                s.EncapsulationSeedSize()] == WANT[bits]


@pytest.mark.parametrize("bits", [384, 521])
def test_entry_points_fail_without_a_device(bits):
    from circl_b200 import _ffi
    if _ffi.lib().cb200_device_count() > 0:
        pytest.skip("a CUDA device is visible")
    m = importlib.import_module(f"circl_b200.p{bits}")
    s, c = m.All()[0], CURVES[bits]
    zk, zp = np.zeros((2, c.nbytes), dtype=np.uint8), np.zeros((2, c.npk), dtype=np.uint8)
    for call in (lambda: s.DeriveKeyPairBatch(zk), lambda: s.EncapsulateBatch(zp, zk), lambda: s.DecapsulateBatch(zk, zp),
                 lambda: s.AuthEncapsulateBatch(zp, zk, zk), lambda: s.AuthDecapsulateBatch(zk, zp, zp),
                 lambda: getattr(m, f"p{bits}_keygen")(zk), lambda: getattr(m, f"p{bits}_shared")(zk, zp)):
        with pytest.raises(_ffi.Cb200Error) as ei:
            call()
        assert ei.value.code == -2 and "not initialised" in str(ei.value)


@pytest.mark.parametrize("bits", [384, 521])
def test_unmarshal_validates_like_crypto_ecdh(bits):
    from circl_b200 import hpke, mlkem
    m = importlib.import_module(f"circl_b200.p{bits}")
    s, c = m.All()[0], CURVES[bits]
    g = enc(c, c.g)
    assert s.UnmarshalBinaryPublicKey(g).MarshalBinary() == g
    for bad in (b"\x02" + g[1:], bytes(c.npk), g[:-1] + bytes([g[-1] ^ 1])):
        with pytest.raises(m.ErrInvalidKEMPublicKey):
            s.UnmarshalBinaryPublicKey(bad)
    with pytest.raises(mlkem.ErrPubKeySize):
        s.UnmarshalBinaryPublicKey(g[:-1])
    top = (c.n - 1).to_bytes(c.nbytes, "big")
    assert s.UnmarshalBinaryPrivateKey(top).MarshalBinary() == top
    bads = [0, c.n, 2**(8 * c.nbytes) - 1] + ([2 << (8 * (c.nbytes - 1))] if bits == 521 else [])
    for bad in bads:
        with pytest.raises(m.ErrInvalidKEMPrivateKey):
            s.UnmarshalBinaryPrivateKey(bad.to_bytes(c.nbytes, "big"))
    with pytest.raises(mlkem.ErrPrivKeySize):
        s.UnmarshalBinaryPrivateKey(bytes(c.nbytes + 1))
    sk = s.UnmarshalBinaryPrivateKey((7).to_bytes(c.nbytes, "big"))
    with pytest.raises(mlkem.ErrPubKeySize):
        s.Decapsulate(sk, bytes(32))
    with pytest.raises(m.ErrInvalidKEMPublicKey):
        s.Decapsulate(sk, bytes(c.npk))
    with pytest.raises(mlkem.ErrSeedSize):
        s.DeriveKeyPair(bytes(c.nbytes + 1))
    with pytest.raises(mlkem.ErrTypeMismatch):
        s.Decapsulate(hpke.All()[0].UnmarshalBinaryPrivateKey(bytes(32)), g)
