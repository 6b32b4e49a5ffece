"""P-521 over the C ABI: the raw ECDH step and the kem.AuthScheme mirror of HPKE's DHKEM(P-521, HKDF-SHA512).

  p521_keygen / p521_shared        crypto/ecdh.P521() PublicKey / ECDH, batched (as circl_b200.p256's)
  HPKE_KEM_P521_HKDF_SHA512        DHKEM(P-521, HKDF-SHA512), kem_id 0x12    hpke/shortkem.go, hpke/kembase.go

circl_b200.p256's code on P-521: sk and seeds 66 bytes, pk and enc 133 (0x04 || X || Y), ss 64.  Keys are validated as
crypto/ecdh does; ErrInvalidKEMPublicKey and ErrInvalidKEMPrivateKey are P-256's classes (the same reference errors)
and carry .status the same way.  Registered here rather than in hpke.All() or p256.All().
"""
from __future__ import annotations

from .p256 import Curve, ErrInvalidKEMPrivateKey, ErrInvalidKEMPublicKey, NistDHKEM, PrivateKey, PublicKey, ecdh

__all__ = ["ByName", "All", "ErrInvalidKEMPublicKey", "ErrInvalidKEMPrivateKey", "p521_keygen", "p521_shared",
           "PrivateKey", "PublicKey"]

P = 2**521 - 1
N = 0x01fffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffa51868783bf2f966b7fcc0148f709a5d03bb5c9b8899c47aebb6fb71e91386409
B = 0x0051953eb9618e1c9a1f929a21a0b68540eea2da725b99b315f3b8b489918ef109e156193951ec7e937b1652c0bd3bb1bf073573df883d2c34f1ef451fd46b503f00
CURVE = Curve("p521", 66, P, N, B)


def p521_keygen(scalars):
    """(n, 66) big-endian scalars in [1, n - 1] -> (n, 133) public keys 0x04 || X || Y.  An invalid scalar raises
    ErrInvalidKEMPrivateKey (with .status) after the batch ran; its row is all zero."""
    return ecdh(CURVE, scalars, None)


def p521_shared(scalars, points):
    """(n, 66) scalars, (n, 133) public keys -> (n, 66) X coordinates of [k]P.  Invalid inputs raise as p521_keygen
    (ErrInvalidKEMPrivateKey before ErrInvalidKEMPublicKey)."""
    return ecdh(CURVE, scalars, points)


_SCHEME = NistDHKEM("HPKE_KEM_P521_HKDF_SHA512", 0x12, 64, CURVE)


def ByName(name: str):
    """kem/schemes/schemes.go:70 -- case-insensitive lookup; None if unknown."""
    return _SCHEME if name.lower() == "hpke_kem_p521_hkdf_sha512" else None


def All():
    return [_SCHEME]
