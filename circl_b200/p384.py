"""P-384 over the C ABI: the raw ECDH step and the kem.AuthScheme mirror of HPKE's DHKEM(P-384, HKDF-SHA384).

  p384_keygen / p384_shared        crypto/ecdh.P384() PublicKey / ECDH, batched (as circl_b200.p256's)
  HPKE_KEM_P384_HKDF_SHA384        DHKEM(P-384, HKDF-SHA384), kem_id 0x11    hpke/shortkem.go, hpke/kembase.go

circl_b200.p256's code on P-384: sk and seeds 48 bytes, pk and enc 97 (0x04 || X || Y), ss 48.  Keys are validated as
crypto/ecdh does; ErrInvalidKEMPublicKey and ErrInvalidKEMPrivateKey are P-256's classes (the same reference errors)
and carry .status the same way.  Registered here rather than in hpke.All() or p256.All().
"""
from __future__ import annotations

from .p256 import Curve, ErrInvalidKEMPrivateKey, ErrInvalidKEMPublicKey, NistDHKEM, PrivateKey, PublicKey, ecdh

__all__ = ["ByName", "All", "ErrInvalidKEMPublicKey", "ErrInvalidKEMPrivateKey", "p384_keygen", "p384_shared",
           "PrivateKey", "PublicKey"]

P = 2**384 - 2**128 - 2**96 + 2**32 - 1
N = 0xffffffffffffffffffffffffffffffffffffffffffffffffc7634d81f4372ddf581a0db248b0a77aecec196accc52973
B = 0xb3312fa7e23ee7e4988e056be3f82d19181d9c6efe8141120314088f5013875ac656398d8a2ed19d2a85c8edd3ec2aef
CURVE = Curve("p384", 48, P, N, B)


def p384_keygen(scalars):
    """(n, 48) big-endian scalars in [1, n - 1] -> (n, 97) public keys 0x04 || X || Y.  An invalid scalar raises
    ErrInvalidKEMPrivateKey (with .status) after the batch ran; its row is all zero."""
    return ecdh(CURVE, scalars, None)


def p384_shared(scalars, points):
    """(n, 48) scalars, (n, 97) public keys -> (n, 48) X coordinates of [k]P.  Invalid inputs raise as p384_keygen
    (ErrInvalidKEMPrivateKey before ErrInvalidKEMPublicKey)."""
    return ecdh(CURVE, scalars, points)


_SCHEME = NistDHKEM("HPKE_KEM_P384_HKDF_SHA384", 0x11, 48, CURVE)


def ByName(name: str):
    """kem/schemes/schemes.go:70 -- case-insensitive lookup; None if unknown."""
    return _SCHEME if name.lower() == "hpke_kem_p384_hkdf_sha384" else None


def All():
    return [_SCHEME]
