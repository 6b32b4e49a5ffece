"""P-256 over the C ABI: the raw ECDH step and the kem.AuthScheme mirror of HPKE's DHKEM(P-256, HKDF-SHA256).
The ECDH step (ecdh) and the scheme class (NistDHKEM) take the curve (Curve) as a parameter; circl_b200.p384 and
circl_b200.p521 use them for P-384 and P-521.  These three names are the package's shared machinery, not part of this
module's public surface.

  p256_keygen / p256_shared        crypto/ecdh.P256() PublicKey / ECDH, batched (like x448.x448_keygen / x448_shared)
  HPKE_KEM_P256_HKDF_SHA256        DHKEM(P-256, HKDF-SHA256), kem_id 0x10    hpke/shortkem.go, hpke/kembase.go

The scheme has the whole surface of circl_b200.hpke.DHKEM (it is one, on the cb200_hpke_p256_* entry points): sk 32
bytes (a big-endian scalar), pk and enc 65 (0x04 || X || Y), seeds 32, ss 32.  Keys are validated as the reference's
UnmarshalBinary* do (crypto/ecdh NewPrivateKey / NewPublicKey).  In a batch, an invalid pkR, enc or pkS raises
ErrInvalidKEMPublicKey and an invalid skR or skS ErrInvalidKEMPrivateKey (the latter first when both occur), for
numpy arrays and CUDA tensors alike; .status holds the per-op flags (bit 0 public, bit 1 private), the failed
operations' secrets are all zero, and the other operations' results are complete.  Registered here rather than in
hpke.All(), which keeps its two Montgomery-curve schemes.
"""
from __future__ import annotations

import os

import numpy as np

from ._ffi import Cb200Error, check, lib
from .hpke import DHKEM, PrivateKey as _DHPrivateKey
from .hybrid import _is_torch, _new, _prep, _ptr, _zeros
from .mlkem import ErrPrivKeySize, ErrPubKeySize, KemError, PublicKey

__all__ = ["P256DHKEM", "ByName", "All", "ErrInvalidKEMPublicKey", "ErrInvalidKEMPrivateKey", "p256_keygen",
           "p256_shared", "PrivateKey", "PublicKey"]


class Curve:
    """A NIST curve y^2 = x^3 - 3x + b mod p of order n, with `size`-byte scalars and coordinates, on the C entry points
    cb200_<prefix> and cb200_hpke_<prefix>_*."""

    def __init__(self, prefix: str, size: int, p: int, n: int, b: int):
        self.prefix, self.size, self.p, self.n, self.b = prefix, size, p, n, b
        self.npk = 1 + 2 * size

    def scalar_ok(self, b: bytes) -> bool:
        return 0 < int.from_bytes(b, "big") < self.n

    def point_ok(self, b: bytes) -> bool:
        if len(b) != self.npk or b[0] != 4:
            return False
        x, y = int.from_bytes(b[1:1 + self.size], "big"), int.from_bytes(b[1 + self.size:], "big")
        return x < self.p and y < self.p and (y * y - (x * x * x - 3 * x + self.b)) % self.p == 0


P = 2**256 - 2**224 + 2**192 + 2**96 - 1
N = 0xffffffff00000000ffffffffffffffffbce6faada7179e84f3b9cac2fc632551
B = 0x5ac635d8aa3a93e7b3ebbd55769886bc651d06b0cc53b0f63bce3c3e27d2604b
CURVE = Curve("p256", 32, P, N, B)


class ErrInvalidKEMPublicKey(KemError):  # hpke.ErrInvalidKEMPublicKey, hpke/hpke.go:278
    pass


class ErrInvalidKEMPrivateKey(KemError):  # hpke.ErrInvalidKEMPrivateKey, hpke/hpke.go:279
    pass


def _err(cls, msg, status):
    e = cls(msg)
    e.status = status
    return e


def _raise_for(code, status):
    """CB200_ERR_PRIVKEY / CB200_ERR_PUBKEY of a host-pointer call, or the status bits of a device-pointer call."""
    if _is_torch(status):
        priv, pub = bool((status & 2).any()), bool((status & 1).any())
    else:
        priv, pub = code == -5, code == -3
    if priv:
        raise _err(ErrInvalidKEMPrivateKey, "hpke: invalid KEM private key", status)
    if pub:
        raise _err(ErrInvalidKEMPublicKey, "hpke: invalid KEM public key", status)


# ---------------------------------------------------------------- the raw ECDH step
def ecdh(curve: Curve, scalars, points):
    """KeyGen (points None) or Shared on `curve`; see p256_keygen / p256_shared."""
    B, W = curve.size, curve.npk
    k = _prep(scalars, B, ValueError(f"scalars: (n, {B}) uint8"))
    n = k.shape[0]
    pt = None
    if points is not None:
        pt = _prep(points, W, ValueError(f"points: (n, {W}) uint8"))
        if pt.shape[0] != n or _is_torch(pt) != _is_torch(k):
            raise ValueError(f"points: (n, {W}) uint8 on the scalars' side")
    out, status = _new(k, (n, W if pt is None else B)), _zeros(k, (n,))
    try:
        check(getattr(lib(), "cb200_" + curve.prefix)(_ptr(k), None if pt is None else _ptr(pt), _ptr(out),
                                                       _ptr(status), n))
    except Cb200Error as e:
        if e.code not in (-3, -5):
            raise
        _raise_for(e.code, status)
    if _is_torch(status) and bool(status.any()):
        _raise_for(0, status)
    return out


def p256_keygen(scalars):
    """(n, 32) big-endian scalars in [1, n - 1] -> (n, 65) public keys 0x04 || X || Y.  An invalid scalar raises
    ErrInvalidKEMPrivateKey (with .status) after the batch ran; its row is all zero."""
    return ecdh(CURVE, scalars, None)


def p256_shared(scalars, points):
    """(n, 32) scalars, (n, 65) public keys -> (n, 32) X coordinates of [k]P.  Invalid inputs raise as p256_keygen
    (ErrInvalidKEMPrivateKey before ErrInvalidKEMPublicKey)."""
    return ecdh(CURVE, scalars, points)


# ---------------------------------------------------------------- DHKEM(P-256, HKDF-SHA256)
class PrivateKey(_DHPrivateKey):
    """kem.PrivateKey of a NIST DHKEM: the big-endian scalar (32 bytes for P-256)."""

    def Public(self) -> PublicKey:
        """KeyGen of this key on the GPU (shortkem.go:151-157)."""
        sk = np.frombuffer(self._packed, dtype=np.uint8).reshape(1, -1)
        return PublicKey(self._scheme, ecdh(self._scheme._curve, sk, None)[0].tobytes())


class NistDHKEM(DHKEM):
    """A NIST DHKEM (kem_id `ident`, shared secrets of `nss` bytes) on the cb200_hpke_<curve.prefix>_* entry points;
    P256DHKEM below, and circl_b200.p384 / p521's schemes."""

    _Priv = PrivateKey

    def __init__(self, name, ident, nss, curve):
        super().__init__(name, ident, curve.size, nss)
        self._curve = curve
        self._npk = curve.npk

    def _c(self, name, *args):
        """cb200_hpke_<prefix>_<name>(args...)"""
        return getattr(lib(), f"cb200_hpke_{self._curve.prefix}_" + name)(*args)

    @staticmethod
    def _run(call, status):
        try:
            check(call())
        except Cb200Error as e:
            if e.code not in (-3, -5):
                raise
            _raise_for(e.code, status)
        if _is_torch(status) and bool(status.any()):
            _raise_for(0, status)

    def UnmarshalBinaryPublicKey(self, buf: bytes) -> PublicKey:
        """shortkem.go:115-130: the size, then crypto/ecdh NewPublicKey (0x04 || X || Y, X, Y < p, on the curve)."""
        pk = super().UnmarshalBinaryPublicKey(buf)
        if not self._curve.point_ok(bytes(buf)):
            raise _err(ErrInvalidKEMPublicKey, "hpke: invalid KEM public key", None)
        return pk

    def UnmarshalBinaryPrivateKey(self, buf: bytes) -> PrivateKey:
        """shortkem.go:103-113: the size, then crypto/ecdh NewPrivateKey (0 < k < n)."""
        sk = super().UnmarshalBinaryPrivateKey(buf)
        if not self._curve.scalar_ok(bytes(buf)):
            raise _err(ErrInvalidKEMPrivateKey, "hpke: invalid KEM private key", None)
        return sk

    def GenerateKeyPair(self):
        """A random scalar in [1, n - 1] (crypto/ecdh GenerateKey, shortkem.go:92-100)."""
        while True:
            b = bytearray(os.urandom(self._nsk))
            b[0] &= (1 << (self._curve.n.bit_length() - 8 * (self._nsk - 1))) - 1  # P-521: the top byte's one bit
            b = bytes(b)
            if self._curve.scalar_ok(b):
                sk = PrivateKey(self, b)
                return sk.Public(), sk


class P256DHKEM(NistDHKEM):
    """DHKEM(P-256, HKDF-SHA256) on the cb200_hpke_p256_* entry points."""

    def __init__(self):
        super().__init__("HPKE_KEM_P256_HKDF_SHA256", 0x10, 32, CURVE)


_SCHEME = P256DHKEM()


def ByName(name: str):
    """kem/schemes/schemes.go:70 -- case-insensitive lookup; None if unknown."""
    return _SCHEME if name.lower() == "hpke_kem_p256_hkdf_sha256" else None


def All():
    return [_SCHEME]
