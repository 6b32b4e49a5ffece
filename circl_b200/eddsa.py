"""sign.Scheme mirrors for Ed25519 (sign/ed25519/signapi.go) and Ed25519-Dilithium2 (sign/eddilithium2/signapi.go)
over the C ABI.

Same method names and errors as `mldsa.Scheme`.  Both schemes are pure: neither takes a context string
(SupportsContext() is False, a non-empty context raises ErrContextNotSupported).  They are registered here rather
than in `mldsa.All()`, which keeps the lattice family.
"""
from __future__ import annotations

import os

import numpy as np

from ._ffi import check, lib
from .mldsa import ErrContextNotSupported, ErrPrivKeySize, ErrPubKeySize, PrivateKey, PublicKey, SignatureOpts

__all__ = ["Ed25519", "EdDilithium2", "ByName", "All", "SignatureOpts", "ErrContextNotSupported"]


def _messages(messages):
    n = len(messages)
    off = np.zeros(n + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(m) for m in messages], dtype=np.uint64)
    blob = np.frombuffer(b"".join(messages) + b"\0" * 8, dtype=np.uint8)  # 8 bytes of read padding
    return blob, off


class _Scheme:
    _prefix = ""
    _name = ""

    def _size(self, what: str) -> int:
        return int(getattr(lib(), f"cb200_{self._prefix}_{what}_size")())

    def Name(self) -> str:
        return self._name

    def PublicKeySize(self) -> int:
        return self._size("public_key")

    def PrivateKeySize(self) -> int:
        return self._size("private_key")

    def SignatureSize(self) -> int:
        return self._size("signature")

    def SeedSize(self) -> int:
        return self._size("seed")

    def SupportsContext(self) -> bool:
        return False

    def UnmarshalBinaryPrivateKey(self, buf: bytes) -> PrivateKey:
        if len(buf) != self.PrivateKeySize():
            raise ErrPrivKeySize("sign: invalid private key size")
        return PrivateKey(self, buf)

    def UnmarshalBinaryPublicKey(self, buf: bytes) -> PublicKey:
        if len(buf) != self.PublicKeySize():
            raise ErrPubKeySize("sign: invalid public key size")
        return PublicKey(self, buf)

    def DeriveKey(self, seed: bytes):
        if len(seed) != self.SeedSize():
            raise ValueError("sign: invalid seed size")  # the reference panics with sign.ErrSeedSize
        pk, sk = self.DeriveKeyBatch(np.frombuffer(seed, dtype=np.uint8).reshape(1, -1))
        return PublicKey(self, pk[0].tobytes()), PrivateKey(self, sk[0].tobytes())

    def GenerateKey(self):
        return self.DeriveKey(os.urandom(self.SeedSize()))

    def DeriveKeyBatch(self, seeds):
        """seeds: (n, 32) uint8 -> (pk (n, PublicKeySize), sk (n, PrivateKeySize))."""
        seeds = np.ascontiguousarray(seeds, dtype=np.uint8)
        if seeds.ndim != 2 or seeds.shape[1] != self.SeedSize():
            raise ValueError("sign: invalid seed size")
        n = seeds.shape[0]
        pk = np.empty((n, self.PublicKeySize()), dtype=np.uint8)
        sk = np.empty((n, self.PrivateKeySize()), dtype=np.uint8)
        check(getattr(lib(), f"cb200_{self._prefix}_keygen")(seeds.ctypes.data, pk.ctypes.data, sk.ctypes.data, n))
        return pk, sk

    def _keys(self, keys, n, size, cls, err):
        if isinstance(keys, cls):
            if len(keys._packed) != size:  # a key of another scheme: the C call would read `size` bytes of it
                raise err("sign: invalid key size")
            return np.frombuffer(keys._packed, dtype=np.uint8), 0
        k = np.ascontiguousarray(keys, dtype=np.uint8)
        if k.shape != (n, size):
            raise err("sign: invalid key size")
        return k, size

    def Sign(self, sk: PrivateKey, message: bytes, opts: SignatureOpts | None = None) -> bytes:
        if not isinstance(sk, PrivateKey):
            raise TypeError("sign: wrong private key type")  # the reference panics with sign.ErrTypeMismatch
        ctx = opts.Context if opts is not None else b""
        return self.SignBatch(sk, [message], ctx=ctx)[0].tobytes()

    def Verify(self, pk: PublicKey, message: bytes, signature: bytes, opts: SignatureOpts | None = None) -> bool:
        if not isinstance(pk, PublicKey):
            raise TypeError("sign: wrong public key type")
        ctx = opts.Context if opts is not None else b""
        if ctx:
            raise ErrContextNotSupported("sign: context not supported")
        if len(signature) != self.SignatureSize():
            return False
        return bool(self.VerifyBatch(pk, [message], np.frombuffer(signature, dtype=np.uint8).reshape(1, -1))[0])

    def VerifyBatch(self, pks, messages, sigs, ctx: bytes = b""):
        """pks: one PublicKey (shared) or (n, PublicKeySize) uint8; sigs: (n, SignatureSize) uint8 -> (n,) bool."""
        if ctx:
            raise ErrContextNotSupported("sign: context not supported")
        n = len(messages)
        pk, stride = self._keys(pks, n, self.PublicKeySize(), PublicKey, ErrPubKeySize)
        sigs = np.ascontiguousarray(sigs, dtype=np.uint8)
        if sigs.shape != (n, self.SignatureSize()):
            raise ValueError("sign: signatures must be (n, SignatureSize)")
        blob, off = _messages(messages)
        ok = np.zeros((n,), dtype=np.uint8)
        check(getattr(lib(), f"cb200_{self._prefix}_verify")(pk.ctypes.data, stride, blob.ctypes.data, off.ctypes.data,
                                                              sigs.ctypes.data, ok.ctypes.data, n))
        return ok.astype(bool)


class Ed25519(_Scheme):
    """sign/ed25519 as a sign.Scheme (signapi.go): pure Ed25519, private key = seed || public key."""

    _prefix, _name = "ed25519", "Ed25519"

    def SignBatch(self, sks, messages, ctx: bytes = b""):
        """sks: one PrivateKey (shared) or (n, 64) uint8.  The public half of each key is used as given."""
        if ctx:
            raise ErrContextNotSupported("sign: context not supported")
        n = len(messages)
        sk, stride = self._keys(sks, n, 64, PrivateKey, ErrPrivKeySize)
        blob, off = _messages(messages)
        sig = np.empty((n, 64), dtype=np.uint8)
        check(lib().cb200_ed25519_sign(sk.ctypes.data, stride, blob.ctypes.data, off.ctypes.data, sig.ctypes.data, n))
        return sig


class EdDilithium2(_Scheme):
    """sign/eddilithium2 as a sign.Scheme (signapi.go): Dilithium2 || Ed25519, both halves must verify."""

    _prefix, _name = "eddilithium2", "Ed25519-Dilithium2"

    def SignBatch(self, sks, messages, ctx: bytes = b"", status=None):
        """sks: one PrivateKey (shared) or (n, 2560) uint8.  status: optional (n,) uint8 array receiving the per-op
        576-attempt flags of the Dilithium2 half."""
        if ctx:
            raise ErrContextNotSupported("sign: context not supported")
        n = len(messages)
        sk, stride = self._keys(sks, n, self.PrivateKeySize(), PrivateKey, ErrPrivKeySize)
        blob, off = _messages(messages)
        sig = np.empty((n, self.SignatureSize()), dtype=np.uint8)
        st = status if status is not None else np.zeros((n,), dtype=np.uint8)
        check(lib().cb200_eddilithium2_sign(sk.ctypes.data, stride, blob.ctypes.data, off.ctypes.data, sig.ctypes.data,
                                            st.ctypes.data, n))
        return sig


_SCHEMES = {"ed25519": Ed25519(), "ed25519-dilithium2": EdDilithium2()}


def ByName(name: str):
    """sign/schemes/schemes.go:69 -- case-insensitive lookup; None if unknown."""
    return _SCHEMES.get(name.lower())


def All():
    """In the order of sign/schemes/schemes.go:31-35."""
    return list(_SCHEMES.values())
