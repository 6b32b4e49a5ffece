"""kem.Scheme mirror for FrodoKEM-640-SHAKE (kem/frodo/frodo640shake), over the C ABI.

Same method names, argument meaning and errors as the reference.  The *Batch methods take (n, size) uint8 numpy arrays
(host) or CUDA torch tensors (device), or one key object shared by the batch: then A and H(pk) are computed once per
call and S'A runs as one tensor-core GEMM over the batch.  Decapsulation never fails (implicit rejection), and keys are
not validated, as in the reference.  The scheme is registered here rather than in `mlkem.All()`, `hybrid.All()`,
`x448.All()` or `hpke.All()`, which keep their families.
"""
from __future__ import annotations

import os

import numpy as np

from ._ffi import check, lib
from .hybrid import _is_torch, _new, _prep, _ptr
from .mlkem import (ErrCiphertextSize, ErrPrivKeySize, ErrPubKeySize, ErrSeedSize, ErrTypeMismatch,
                    PrivateKey as _PrivateKey, PublicKey)

__all__ = ["Scheme", "ByName", "All", "PublicKey", "PrivateKey"]

PK, SK, CT, SS, SEED, ESEED = 9616, 19888, 9720, 16, 48, 16


class PrivateKey(_PrivateKey):
    """kem.PrivateKey: s || pk || S^T || H(pk) (frodo.go:334-354)."""

    def Public(self) -> PublicKey:
        """The public key embedded in the private key (frodo.go:466-468)."""
        return PublicKey(self._scheme, self._packed[16:16 + PK])


class FrodoKEM:
    def Name(self) -> str: return "FrodoKEM-640-SHAKE"
    def PublicKeySize(self): return PK
    def PrivateKeySize(self): return SK
    def CiphertextSize(self): return CT
    def SeedSize(self): return SEED
    def EncapsulationSeedSize(self): return ESEED
    def SharedKeySize(self): return SS

    # ---------------------------------------------------------------- single operations
    def UnmarshalBinaryPublicKey(self, buf: bytes) -> PublicKey:
        if len(buf) != PK:
            raise ErrPubKeySize("kem: invalid public key size")
        return PublicKey(self, buf)

    def UnmarshalBinaryPrivateKey(self, buf: bytes) -> PrivateKey:
        if len(buf) != SK:
            raise ErrPrivKeySize("kem: invalid private key size")
        return PrivateKey(self, buf)

    def GenerateKeyPair(self):
        return self.DeriveKeyPair(os.urandom(SEED))

    def DeriveKeyPair(self, seed: bytes):
        if len(seed) != SEED:
            raise ErrSeedSize("kem: invalid seed size")  # the reference panics with kem.ErrSeedSize
        pk, sk = self.DeriveKeyPairBatch(_row(seed))
        return PublicKey(self, pk[0].tobytes()), PrivateKey(self, sk[0].tobytes())

    def Encapsulate(self, pk: PublicKey):
        self._check(pk, PublicKey)
        return self.EncapsulateDeterministically(pk, os.urandom(ESEED))

    # Argument checks in the reference's order: the seed or ciphertext length first, then the key type
    # (frodo.go:499-529).
    def EncapsulateDeterministically(self, pk: PublicKey, seed: bytes):
        if len(seed) != ESEED:
            raise ErrSeedSize("kem: invalid seed size")
        self._check(pk, PublicKey)
        ct, ss = self.EncapsulateBatch(pk, _row(seed))
        return ct[0].tobytes(), ss[0].tobytes()

    def Decapsulate(self, sk: PrivateKey, ct: bytes) -> bytes:
        if len(ct) != CT:
            raise ErrCiphertextSize("kem: invalid ciphertext size")
        self._check(sk, PrivateKey)
        return self.DecapsulateBatch(sk, _row(ct))[0].tobytes()

    # ---------------------------------------------------------------- batches
    def DeriveKeyPairBatch(self, seeds):
        """(n, 48) seeds -> (pk (n, 9616), sk (n, 19888))."""
        s = _prep(seeds, SEED, ErrSeedSize("kem: invalid seed size"))
        n = s.shape[0]
        pk, sk = _new(s, (n, PK)), _new(s, (n, SK))
        check(lib().cb200_frodo640shake_keygen(_ptr(s), _ptr(pk), _ptr(sk), n))
        return pk, sk

    def EncapsulateBatch(self, pks, seeds):
        """pks: one PublicKey (shared) or (n, 9616); seeds (n, 16) -> (ct (n, 9720), ss (n, 16))."""
        es = _prep(seeds, ESEED, ErrSeedSize("kem: invalid seed size"))
        n = es.shape[0]
        pk, stride = self._keys(pks, PublicKey, PK, n, es, ErrPubKeySize("kem: invalid public key size"))
        ct, ss = _new(es, (n, CT)), _new(es, (n, SS))
        check(lib().cb200_frodo640shake_encaps(_ptr(pk), stride, _ptr(es), _ptr(ct), _ptr(ss), n))
        return ct, ss

    def DecapsulateBatch(self, sks, cts):
        """sks: one PrivateKey (shared) or (n, 19888); cts (n, 9720) -> ss (n, 16)."""
        c = _prep(cts, CT, ErrCiphertextSize("kem: invalid ciphertext size"))
        n = c.shape[0]
        sk, stride = self._keys(sks, PrivateKey, SK, n, c, ErrPrivKeySize("kem: invalid private key size"))
        ss = _new(c, (n, SS))
        check(lib().cb200_frodo640shake_decaps(_ptr(sk), stride, _ptr(c), _ptr(ss), n))
        return ss

    # ---------------------------------------------------------------- helpers
    def _check(self, key, cls):
        if not isinstance(key, cls) or key._scheme is not self:
            raise ErrTypeMismatch("kem: type mismatch")

    def _keys(self, keys, cls, width, n, like, err):
        """One key object (shared by the batch) or an (n, width) array -> (array, stride)."""
        if isinstance(keys, (PublicKey, _PrivateKey)):
            self._check(keys, cls)
            arr = _row(keys._packed)
            if _is_torch(like):
                import torch
                arr = torch.from_numpy(arr.copy()).to(like.device)
            return arr, 0
        arr = _prep(keys, width, err)
        if arr.shape[0] != n:
            raise err
        return arr, width


def _row(b: bytes):
    return np.frombuffer(bytes(b), dtype=np.uint8).reshape(1, -1)


_SCHEME = FrodoKEM()


def Scheme() -> FrodoKEM:
    """frodo640shake.Scheme()."""
    return _SCHEME


def ByName(name: str):
    """kem/schemes/schemes.go:70 -- case-insensitive lookup; None if unknown."""
    return _SCHEME if name.lower() == "frodokem-640-shake" else None


def All():
    return [_SCHEME]
