"""kem.Scheme / kem.AuthScheme mirrors for HPKE's two Montgomery-curve DHKEMs, over the C ABI:

  HPKE_KEM_X25519_HKDF_SHA256   DHKEM(X25519, HKDF-SHA256), kem_id 0x20    hpke/xkem.go, hpke/kembase.go
  HPKE_KEM_X448_HKDF_SHA512     DHKEM(X448, HKDF-SHA512),   kem_id 0x21    (kem/schemes/schemes.go:35-55)

Same method names, argument meaning and errors as the reference.  Besides kem.Scheme, a DHKEM has
AuthEncapsulate / AuthEncapsulateDeterministically / AuthDecapsulate (kem/kem.go:84-90).  The *Batch methods take
(n, size) uint8 numpy arrays (host) or CUDA torch tensors (device), or one key object shared by the batch.  A DH step
with a low-order point raises ErrInvalidKEMSharedSecret (hpke.ErrInvalidKEMSharedSecret), on the host and on the device
path alike (the device path reads the status array back, which waits for the call): its .status holds the per-op
flags, the failed operations' secrets are all zero and must not be used, and the other operations' results are
complete.  These schemes are registered here rather than in `hybrid.All()` or `x448.All()`, which keep their
families.
"""
from __future__ import annotations

import os

import numpy as np

from ._ffi import Cb200Error, check, lib
from .hybrid import _is_torch, _new, _prep, _ptr, _zeros
from .mlkem import (ErrPrivKeySize, ErrPubKeySize, ErrSeedSize, ErrTypeMismatch, KemError, PrivateKey as _PrivateKey,
                    PublicKey)

__all__ = ["DHKEM", "ByName", "All", "ErrInvalidKEMSharedSecret", "PublicKey", "PrivateKey"]


class ErrInvalidKEMSharedSecret(KemError):  # hpke.ErrInvalidKEMSharedSecret, hpke/hpke.go:280
    pass


class PrivateKey(_PrivateKey):
    """kem.PrivateKey of a DHKEM: the private key as stored (unclamped)."""

    def Public(self) -> PublicKey:
        """KeyGen of this key on the GPU (xkem.go:146-163)."""
        s = self._scheme
        sk = np.frombuffer(self._packed, dtype=np.uint8).reshape(1, -1)
        pk = np.empty_like(sk)
        check((lib().cb200_x25519 if s._n == 32 else lib().cb200_x448)(_ptr(sk), None, _ptr(pk), None, 1))
        return PublicKey(s, pk[0].tobytes())


def _invalid(status):
    err = ErrInvalidKEMSharedSecret("hpke: invalid KEM shared secret")
    err.status = status
    return err


def _run(call, status):
    """Runs one batched call.  A host-pointer call reports failed operations as CB200_ERR_PUBKEY; a device-pointer call
    only through status, which is read here so that a failure is never silent (an all-zero secret is public)."""
    try:
        check(call())
    except Cb200Error as e:
        if e.code != -3:
            raise
        raise _invalid(status) from None
    if _is_torch(status) and bool(status.any()):
        raise _invalid(status)


class DHKEM:
    """One of the two DHKEMs; the sizes follow from the id (xkem.go:20-24, kembase.go:34).  A subclass with other
    key sizes (_nsk, _npk), its own entry points (_c), key class (_Priv) and errors (_run) is circl_b200.p256's."""

    _Priv = PrivateKey

    def __init__(self, name: str, ident: int, n: int, nss: int):
        self._name, self._id, self._n, self._nss = name, ident, n, nss
        self._nsk = self._npk = n

    def Name(self) -> str: return self._name
    def PublicKeySize(self): return self._npk
    def PrivateKeySize(self): return self._nsk
    def CiphertextSize(self): return self._npk
    def SeedSize(self): return self._nsk
    def EncapsulationSeedSize(self): return self._nsk
    def SharedKeySize(self): return self._nss

    def _c(self, name, *args):
        """cb200_hpke_<name>(id, args...)"""
        return getattr(lib(), "cb200_hpke_" + name)(self._id, *args)

    @staticmethod
    def _run(call, status):
        _run(call, status)

    # ---------------------------------------------------------------- single operations
    def UnmarshalBinaryPublicKey(self, buf: bytes) -> PublicKey:
        if len(buf) != self._npk:
            raise ErrPubKeySize("kem: invalid public key size")
        return PublicKey(self, buf)

    def UnmarshalBinaryPrivateKey(self, buf: bytes) -> PrivateKey:
        if len(buf) != self._nsk:
            raise ErrPrivKeySize("kem: invalid private key size")
        return self._Priv(self, buf)

    def GenerateKeyPair(self):
        """A random private key, as the reference draws it (xkem.go:73-80)."""
        sk = self._Priv(self, os.urandom(self._nsk))
        return sk.Public(), sk

    # Argument checks in the reference's order: the seed (DeriveKeyPair of the ephemeral key) or the encapsulation
    # (parsed as a public key) first, then the key types (calcDH's type assertion).
    def DeriveKeyPair(self, seed: bytes):
        self._seed(seed)  # the reference panics with kem.ErrSeedSize
        pk, sk = self.DeriveKeyPairBatch(self._row(seed))
        return PublicKey(self, pk[0].tobytes()), self._Priv(self, sk[0].tobytes())

    def Encapsulate(self, pk: PublicKey):
        return self.EncapsulateDeterministically(pk, os.urandom(self._nsk))

    def EncapsulateDeterministically(self, pk: PublicKey, seed: bytes):
        self._seed(seed)
        self._check(pk, PublicKey)
        enc, ss = self.EncapsulateBatch(pk, self._row(seed))
        return enc[0].tobytes(), ss[0].tobytes()

    def Decapsulate(self, sk: PrivateKey, ct: bytes) -> bytes:
        self.UnmarshalBinaryPublicKey(ct)  # ct is parsed as a public key: kem.ErrPubKeySize (kembase.go:222)
        self._check(sk, PrivateKey)
        return self.DecapsulateBatch(sk, self._row(ct))[0].tobytes()

    def AuthEncapsulate(self, pkr: PublicKey, sks: PrivateKey):
        return self.AuthEncapsulateDeterministically(pkr, sks, os.urandom(self._nsk))

    def AuthEncapsulateDeterministically(self, pkr: PublicKey, sks: PrivateKey, seed: bytes):
        self._seed(seed)
        self._check(pkr, PublicKey)
        self._check(sks, PrivateKey)
        enc, ss = self.AuthEncapsulateBatch(pkr, sks, self._row(seed))
        return enc[0].tobytes(), ss[0].tobytes()

    def AuthDecapsulate(self, skr: PrivateKey, ct: bytes, pks: PublicKey) -> bytes:
        self.UnmarshalBinaryPublicKey(ct)
        self._check(skr, PrivateKey)
        self._check(pks, PublicKey)
        return self.AuthDecapsulateBatch(skr, self._row(ct), pks)[0].tobytes()

    # ---------------------------------------------------------------- batches
    def DeriveKeyPairBatch(self, seeds):
        """(n, N) seeds -> (pk (n, N), sk (n, N))."""
        s = _prep(seeds, self._nsk, ErrSeedSize("kem: invalid seed size"))
        n = s.shape[0]
        pk, sk = _new(s, (n, self._npk)), _new(s, (n, self._nsk))
        check(self._c("keygen", _ptr(s), _ptr(pk), _ptr(sk), n))
        return pk, sk

    def EncapsulateBatch(self, pks, seeds):
        """pks: one PublicKey (shared) or (n, N); seeds (n, N) -> (enc (n, N), ss (n, SharedKeySize))."""
        return self._encaps(pks, None, seeds)

    def AuthEncapsulateBatch(self, pkrs, skss, seeds):
        """pkrs / skss: one key object (shared) or (n, N) each."""
        return self._encaps(pkrs, skss, seeds)

    def DecapsulateBatch(self, sks, encs):
        """sks: one PrivateKey (shared; its public key is computed once) or (n, N); encs (n, N) -> ss."""
        return self._decaps(sks, encs, None)

    def AuthDecapsulateBatch(self, skrs, encs, pkss):
        return self._decaps(skrs, encs, pkss)

    def _encaps(self, pkrs, skss, seeds):
        es = _prep(seeds, self._nsk, ErrSeedSize("kem: invalid seed size"))
        n = es.shape[0]
        pk, pks = self._keys(pkrs, PublicKey, n, es, ErrPubKeySize("kem: invalid public key size"))
        enc, ss, status = _new(es, (n, self._npk)), _new(es, (n, self._nss)), _zeros(es, (n,))
        if skss is None:
            self._run(lambda: self._c("encaps", _ptr(pk), pks, _ptr(es), _ptr(enc), _ptr(ss), _ptr(status), n), status)
        else:
            sk, sks = self._keys(skss, PrivateKey, n, es, ErrPrivKeySize("kem: invalid private key size"))
            self._run(lambda: self._c("auth_encaps", _ptr(pk), pks, _ptr(sk), sks, _ptr(es), _ptr(enc), _ptr(ss),
                                      _ptr(status), n), status)
        return enc, ss

    def _decaps(self, skrs, encs, pkss):
        c = _prep(encs, self._npk, ErrPubKeySize("kem: invalid public key size"))
        n = c.shape[0]
        sk, sks = self._keys(skrs, PrivateKey, n, c, ErrPrivKeySize("kem: invalid private key size"))
        ss, status = _new(c, (n, self._nss)), _zeros(c, (n,))
        if pkss is None:
            self._run(lambda: self._c("decaps", _ptr(sk), sks, _ptr(c), _ptr(ss), _ptr(status), n), status)
        else:
            pk, pks = self._keys(pkss, PublicKey, n, c, ErrPubKeySize("kem: invalid public key size"))
            self._run(lambda: self._c("auth_decaps", _ptr(sk), sks, _ptr(c), _ptr(pk), pks, _ptr(ss), _ptr(status), n),
                      status)
        return ss

    # ---------------------------------------------------------------- helpers
    def _check(self, key, cls):
        if not isinstance(key, cls) or key._scheme is not self:
            raise ErrTypeMismatch("kem: type mismatch")

    def _seed(self, seed):
        if len(seed) != self._nsk:
            raise ErrSeedSize("kem: invalid seed size")

    @staticmethod
    def _row(b: bytes):
        return np.frombuffer(bytes(b), dtype=np.uint8).reshape(1, -1)

    def _keys(self, keys, cls, n, like, err):
        """One key object (shared by the batch) or an (n, N) array -> (array, stride)."""
        if isinstance(keys, (PublicKey, _PrivateKey)):
            if not isinstance(keys, cls) or keys._scheme is not self:
                raise ErrTypeMismatch("kem: type mismatch")
            arr = self._row(keys._packed)
            if _is_torch(like):
                import torch
                arr = torch.from_numpy(arr.copy()).to(like.device)
            return arr, 0
        width = self._npk if cls is PublicKey else self._nsk
        arr = _prep(keys, width, err)
        if arr.shape[0] != n:
            raise err
        return arr, width


_SCHEMES = {"hpke_kem_x25519_hkdf_sha256": DHKEM("HPKE_KEM_X25519_HKDF_SHA256", 0x20, 32, 32),
            "hpke_kem_x448_hkdf_sha512": DHKEM("HPKE_KEM_X448_HKDF_SHA512", 0x21, 56, 64)}


def ByName(name: str):
    """kem/schemes/schemes.go:70 -- case-insensitive lookup; None if unknown."""
    return _SCHEMES.get(name.lower())


def All():
    """In the order of kem/schemes/schemes.go:35-55 (X25519, then X448)."""
    return list(_SCHEMES.values())
