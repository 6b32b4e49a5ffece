"""dh/x448 and the kem/hybrid schemes over X448, over the C ABI:

  x448_keygen / x448_shared                dh/x448/key.go:33-46
  Kyber768-X448, Kyber1024-X448            kem/hybrid/hybrid.go:83-93 over kem/hybrid/xkem.go

The two schemes are `hybrid.Hybrid` objects (ids 3 and 4 of include/circl_b200.h); they are registered here rather
than in `hybrid.All()`, which keeps the X25519 family.
"""
from __future__ import annotations

from ._ffi import Cb200Error, check, lib
from .hybrid import Hybrid, _new, _prep, _ptr, _zeros


def x448_keygen(secrets):
    """x448.KeyGen on every row: (n, 56) -> (n, 56) public keys."""
    k = _prep(secrets, 56, ValueError("x448: keys are 56 bytes"))
    out = _new(k, (k.shape[0], 56))
    check(lib().cb200_x448(_ptr(k), None, _ptr(out), None, k.shape[0]))
    return out


def x448_shared(secrets, publics):
    """x448.Shared on every row -> (shared (n, 56), ok (n,) bool); ok False = low-order point, shared all zero."""
    k = _prep(secrets, 56, ValueError("x448: keys are 56 bytes"))
    p = _prep(publics, 56, ValueError("x448: keys are 56 bytes"))
    n = k.shape[0]
    out, status = _new(k, (n, 56)), _zeros(k, (n,))
    try:
        check(lib().cb200_x448(_ptr(k), _ptr(p), _ptr(out), _ptr(status), n))
    except Cb200Error as e:
        if e.code != -3:
            raise
    return out, status == 0


_SCHEMES = {"kyber768-x448": Hybrid("Kyber768-X448", 3), "kyber1024-x448": Hybrid("Kyber1024-X448", 4)}


def ByName(name: str):
    """kem/schemes/schemes.go:70 -- case-insensitive lookup; None if unknown."""
    return _SCHEMES.get(name.lower())


def All():
    return list(_SCHEMES.values())
