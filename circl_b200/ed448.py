"""sign.Scheme mirrors for Ed448 (sign/ed448/signapi.go) and Ed448-Dilithium3 (sign/eddilithium3/signapi.go) over the
C ABI.

Same method names and errors as `mldsa.Scheme`.  Ed448 takes a context string of up to 255 bytes, shared by a batch
(SupportsContext() is True): signing with a longer one raises ErrContextTooLong, verifying with one returns False.
Ed448-Dilithium3 is pure (a non-empty context raises ErrContextNotSupported).  Both are registered here rather than
in `eddsa.All()` or `mldsa.All()`, which keep their families.
"""
from __future__ import annotations

import numpy as np

from ._ffi import check, lib
from .eddsa import _messages, _Scheme
from .mldsa import (ErrContextNotSupported, ErrContextTooLong, ErrPrivKeySize, ErrPubKeySize, PrivateKey, PublicKey,
                    SignatureOpts)

__all__ = ["Ed448", "EdDilithium3", "ByName", "All", "SignatureOpts", "ErrContextNotSupported", "ErrContextTooLong"]

_MAX_CONTEXT = 255


def _ctx(ctx: bytes):
    c = np.frombuffer(bytes(ctx) or b"\0", dtype=np.uint8)
    return c, len(ctx)


class Ed448(_Scheme):
    """sign/ed448 as a sign.Scheme (signapi.go): pure Ed448, private key = seed || public key."""

    _prefix, _name = "ed448", "Ed448"

    def SupportsContext(self) -> bool:
        return True

    def SignBatch(self, sks, messages, ctx: bytes = b""):
        """sks: one PrivateKey (shared) or (n, 114) uint8.  The public half of each key is used as given."""
        if len(ctx) > _MAX_CONTEXT:
            raise ErrContextTooLong("sign: context too long")  # the reference panics
        n = len(messages)
        sk, stride = self._keys(sks, n, 114, PrivateKey, ErrPrivKeySize)
        blob, off = _messages(messages)
        c, clen = _ctx(ctx)
        sig = np.empty((n, 114), dtype=np.uint8)
        check(lib().cb200_ed448_sign(sk.ctypes.data, stride, blob.ctypes.data, off.ctypes.data, c.ctypes.data, clen,
                                     sig.ctypes.data, n))
        return sig

    def Verify(self, pk: PublicKey, message: bytes, signature: bytes, opts: SignatureOpts | None = None) -> bool:
        if not isinstance(pk, PublicKey):
            raise TypeError("sign: wrong public key type")
        ctx = opts.Context if opts is not None else b""
        if len(signature) != self.SignatureSize():
            return False
        return bool(self.VerifyBatch(pk, [message], np.frombuffer(signature, dtype=np.uint8).reshape(1, -1), ctx)[0])

    def VerifyBatch(self, pks, messages, sigs, ctx: bytes = b""):
        """pks: one PublicKey (shared) or (n, 57) uint8; sigs: (n, 114) uint8 -> (n,) bool.  A context over 255 bytes
        verifies nothing."""
        n = len(messages)
        pk, stride = self._keys(pks, n, 57, PublicKey, ErrPubKeySize)
        sigs = np.ascontiguousarray(sigs, dtype=np.uint8)
        if sigs.shape != (n, 114):
            raise ValueError("sign: signatures must be (n, SignatureSize)")
        blob, off = _messages(messages)
        c, clen = _ctx(ctx)
        ok = np.zeros((n,), dtype=np.uint8)
        check(lib().cb200_ed448_verify(pk.ctypes.data, stride, blob.ctypes.data, off.ctypes.data, c.ctypes.data, clen,
                                       sigs.ctypes.data, ok.ctypes.data, n))
        return ok.astype(bool)


class EdDilithium3(_Scheme):
    """sign/eddilithium3 as a sign.Scheme (signapi.go): Dilithium3 || Ed448, both halves must verify."""

    _prefix, _name = "eddilithium3", "Ed448-Dilithium3"

    def SignBatch(self, sks, messages, ctx: bytes = b"", status=None):
        """sks: one PrivateKey (shared) or (n, 4057) uint8.  status: optional (n,) uint8 array receiving the per-op
        576-attempt flags of the Dilithium3 half."""
        if ctx:
            raise ErrContextNotSupported("sign: context not supported")
        n = len(messages)
        sk, stride = self._keys(sks, n, self.PrivateKeySize(), PrivateKey, ErrPrivKeySize)
        blob, off = _messages(messages)
        sig = np.empty((n, self.SignatureSize()), dtype=np.uint8)
        st = status if status is not None else np.zeros((n,), dtype=np.uint8)
        check(lib().cb200_eddilithium3_sign(sk.ctypes.data, stride, blob.ctypes.data, off.ctypes.data, sig.ctypes.data,
                                            st.ctypes.data, n))
        return sig


_SCHEMES = {"ed448": Ed448(), "ed448-dilithium3": EdDilithium3()}


def ByName(name: str):
    """sign/schemes/schemes.go:69 -- case-insensitive lookup; None if unknown."""
    return _SCHEMES.get(name.lower())


def All():
    """In the order of sign/schemes/schemes.go:31-54 (Ed448, then Ed448-Dilithium3)."""
    return list(_SCHEMES.values())
