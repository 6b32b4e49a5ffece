"""kem.Scheme mirrors for the callers on the wire side of ML-KEM (SURVEY.md 8(f) row 4), over the C ABI:

  X-Wing                                   kem/xwing/scheme.go:1-140, xwing.go
  X25519MLKEM768, Kyber768-X25519,
  Kyber512-X25519                          kem/hybrid/hybrid.go:34-62,197-315 over kem/hybrid/xkem.go
  x25519_keygen / x25519_shared            dh/x25519/key.go:44-56

Same method names, argument meaning and error behaviour as the reference; the *Batch methods take (n, size)
uint8 numpy arrays (host) or CUDA torch tensors (device) and are what a GPU call needs to be worth its launch.
"""
from __future__ import annotations

import numpy as np

from ._ffi import Cb200Error, check, lib
from .mlkem import (ErrCiphertextSize, ErrPrivKey, ErrPrivKeySize, ErrPubKey, ErrPubKeySize, ErrSeedSize, ErrTypeMismatch,
                    PrivateKey, PublicKey)


def _is_torch(x) -> bool:
    return type(x).__module__.startswith("torch")


def _ptr(x):
    return x.data_ptr() if _is_torch(x) else x.ctypes.data


def _new(like, shape):
    if _is_torch(like):
        import torch
        return torch.empty(shape, dtype=torch.uint8, device=like.device)
    return np.empty(shape, dtype=np.uint8)


def _zeros(like, shape):
    if _is_torch(like):
        import torch
        return torch.zeros(shape, dtype=torch.uint8, device=like.device)
    return np.zeros(shape, dtype=np.uint8)


def _prep(x, width, err):
    """(n, width) uint8, contiguous, host numpy or CUDA torch."""
    if _is_torch(x):
        import torch
        if not (x.is_cuda and x.dtype == torch.uint8 and x.is_contiguous() and x.dim() == 2 and x.shape[1] == width):
            raise err
        check(lib().cb200_set_stream(torch.cuda.current_stream().cuda_stream))
        return x
    x = np.ascontiguousarray(x, dtype=np.uint8)
    if x.ndim != 2 or x.shape[1] != width:
        raise err
    return x


def _raise_status(e: Cb200Error, status):
    if e.code == -3:
        err = ErrPubKey("kem: invalid public key")
    elif e.code == -5:
        err = ErrPrivKey("kem: invalid private key")
    else:
        raise e
    err.status = status
    raise err from None


# ---------------------------------------------------------------- dh/x25519
def x25519_keygen(secrets):
    """x25519.KeyGen on every row: (n, 32) -> (n, 32) public keys."""
    k = _prep(secrets, 32, ValueError("x25519: keys are 32 bytes"))
    out = _new(k, (k.shape[0], 32))
    check(lib().cb200_x25519(_ptr(k), None, _ptr(out), None, k.shape[0]))
    return out


def x25519_shared(secrets, publics):
    """x25519.Shared on every row -> (shared (n, 32), ok (n,) bool); ok False = small-order point, shared all zero."""
    k = _prep(secrets, 32, ValueError("x25519: keys are 32 bytes"))
    p = _prep(publics, 32, ValueError("x25519: keys are 32 bytes"))
    n = k.shape[0]
    out, status = _new(k, (n, 32)), _zeros(k, (n,))
    try:
        check(lib().cb200_x25519(_ptr(k), _ptr(p), _ptr(out), _ptr(status), n))
    except Cb200Error as e:
        if e.code != -3:
            raise
    return out, status == 0


# ---------------------------------------------------------------- schemes
class _Base:
    def Name(self) -> str:
        return self._name

    def UnmarshalBinaryPublicKey(self, buf: bytes) -> PublicKey:
        if len(buf) != self.PublicKeySize():
            raise ErrPubKeySize("kem: invalid public key size")
        return PublicKey(self, buf)

    def UnmarshalBinaryPrivateKey(self, buf: bytes) -> PrivateKey:
        if len(buf) != self.PrivateKeySize():
            raise ErrPrivKeySize("kem: invalid private key size")
        return PrivateKey(self, buf)

    def GenerateKeyPair(self):
        import os
        return self.DeriveKeyPair(os.urandom(self.SeedSize()))

    def DeriveKeyPair(self, seed: bytes):
        if len(seed) != self.SeedSize():
            raise ValueError("kem: invalid seed size")  # the reference panics with kem.ErrSeedSize
        pk, sk = self.DeriveKeyPairBatch(np.frombuffer(seed, dtype=np.uint8).reshape(1, -1))
        return PublicKey(self, pk[0].tobytes()), PrivateKey(self, sk[0].tobytes())

    def EncapsulateDeterministically(self, pk: PublicKey, seed: bytes):
        if not isinstance(pk, PublicKey) or pk._scheme is not self:
            raise ErrTypeMismatch("kem: type mismatch")
        if len(seed) != self.EncapsulationSeedSize():
            raise ErrSeedSize("kem: invalid seed size")
        ct, ss = self.EncapsulateBatch(pk, np.frombuffer(seed, dtype=np.uint8).reshape(1, -1))
        return ct[0].tobytes(), ss[0].tobytes()

    def Encapsulate(self, pk: PublicKey):
        import os
        return self.EncapsulateDeterministically(pk, os.urandom(self.EncapsulationSeedSize()))

    def Decapsulate(self, sk: PrivateKey, ct: bytes) -> bytes:
        if not isinstance(sk, PrivateKey) or sk._scheme is not self:
            raise ErrTypeMismatch("kem: type mismatch")
        if len(ct) != self.CiphertextSize():
            raise ErrCiphertextSize("kem: invalid ciphertext size")
        return self.DecapsulateBatch(sk, np.frombuffer(ct, dtype=np.uint8).reshape(1, -1))[0].tobytes()

    def _keys(self, keys, cls, size, n, like, err):
        """One key object (shared by the batch) or an (n, size) array -> (array, stride)."""
        if isinstance(keys, cls):
            if keys._scheme is not self:
                raise ErrTypeMismatch("kem: type mismatch")
            arr = np.frombuffer(keys._packed, dtype=np.uint8).reshape(1, size)
            if _is_torch(like):
                import torch
                arr = torch.from_numpy(arr.copy()).to(like.device)
            return arr, 0
        arr = _prep(keys, size, err)
        if arr.shape[0] != n:
            raise err
        return arr, size


class XWing(_Base):
    """kem/xwing: ML-KEM-768 + X25519 with the SHA3-256 combiner (xwing.go:47-66)."""
    _name = "X-Wing"

    def PublicKeySize(self): return 1216
    def PrivateKeySize(self): return 32
    def SeedSize(self): return 32
    def EncapsulationSeedSize(self): return 64
    def CiphertextSize(self): return 1120
    def SharedKeySize(self): return 32

    def DeriveKeyPairBatch(self, seeds):
        """xwing.DeriveKeyPairPacked on every row: (n, 32) -> (pk (n, 1216), sk (n, 32) = the seeds)."""
        s = _prep(seeds, 32, ValueError("kem: invalid seed size"))
        pk = _new(s, (s.shape[0], 1216))
        check(lib().cb200_xwing_keygen(_ptr(s), _ptr(pk), s.shape[0]))
        return pk, (s.clone() if _is_torch(s) else s.copy())

    def EncapsulateBatch(self, pks, eseeds):
        es = _prep(eseeds, 64, ErrSeedSize("kem: invalid seed size"))
        n = es.shape[0]
        pk, stride = self._keys(pks, PublicKey, 1216, n, es, ErrPubKeySize("kem: invalid public key size"))
        ct, ss, status = _new(es, (n, 1120)), _new(es, (n, 32)), _zeros(es, (n,))
        try:
            check(lib().cb200_xwing_encaps(_ptr(pk), stride, _ptr(es), _ptr(ct), _ptr(ss), _ptr(status), n))
        except Cb200Error as e:
            _raise_status(e, status)
        self._last_status = status
        return ct, ss

    def DecapsulateBatch(self, sks, cts):
        c = _prep(cts, 1120, ErrCiphertextSize("kem: invalid ciphertext size"))
        n = c.shape[0]
        sk, stride = self._keys(sks, PrivateKey, 32, n, c, ErrPrivKeySize("kem: invalid private key size"))
        ss = _new(c, (n, 32))
        check(lib().cb200_xwing_decaps(_ptr(sk), stride, _ptr(c), _ptr(ss), n))
        return ss


class Hybrid(_Base):
    """kem/hybrid.scheme: two KEMs side by side (hybrid.go:76-80)."""

    def __init__(self, name: str, ident: int):
        self._name, self._id = name, ident

    def PublicKeySize(self): return lib().cb200_hybrid_public_key_size(self._id)
    def PrivateKeySize(self): return lib().cb200_hybrid_private_key_size(self._id)
    def CiphertextSize(self): return lib().cb200_hybrid_ciphertext_size(self._id)
    def SeedSize(self): return lib().cb200_hybrid_seed_size(self._id)  # max(first, second), hybrid.go:131-139
    def EncapsulationSeedSize(self): return lib().cb200_hybrid_encapsulation_seed_size(self._id)  # hybrid.go:149-157
    def SharedKeySize(self): return lib().cb200_hybrid_shared_key_size(self._id)  # hybrid.go:141-143

    def DeriveKeyPairBatch(self, seeds):
        s = _prep(seeds, self.SeedSize(), ValueError("kem: invalid seed size"))
        n = s.shape[0]
        pk, sk = _new(s, (n, self.PublicKeySize())), _new(s, (n, self.PrivateKeySize()))
        check(lib().cb200_hybrid_keygen(self._id, _ptr(s), _ptr(pk), _ptr(sk), n))
        return pk, sk

    def EncapsulateBatch(self, pks, seeds):
        es = _prep(seeds, self.EncapsulationSeedSize(), ErrSeedSize("kem: invalid seed size"))
        n = es.shape[0]
        pk, stride = self._keys(pks, PublicKey, self.PublicKeySize(), n, es, ErrPubKeySize("kem: invalid public key size"))
        ct, ss, status = _new(es, (n, self.CiphertextSize())), _new(es, (n, self.SharedKeySize())), _zeros(es, (n,))
        try:
            check(lib().cb200_hybrid_encaps(self._id, _ptr(pk), stride, _ptr(es), _ptr(ct), _ptr(ss), _ptr(status), n))
        except Cb200Error as e:
            _raise_status(e, status)
        self._last_status = status
        return ct, ss

    def DecapsulateBatch(self, sks, cts):
        c = _prep(cts, self.CiphertextSize(), ErrCiphertextSize("kem: invalid ciphertext size"))
        n = c.shape[0]
        sksz = self.PrivateKeySize()
        sk, stride = self._keys(sks, PrivateKey, sksz, n, c, ErrPrivKeySize("kem: invalid private key size"))
        if stride == 0:  # the decapsulation flows take one key per operation
            sk = sk.repeat(n, 1) if _is_torch(sk) else np.repeat(sk, n, axis=0)
        ss, status = _new(c, (n, self.SharedKeySize())), _zeros(c, (n,))
        try:
            check(lib().cb200_hybrid_decaps(self._id, _ptr(sk), sksz, _ptr(c), _ptr(ss), _ptr(status), n))
        except Cb200Error as e:
            _raise_status(e, status)
        self._last_status = status
        return ss


_SCHEMES = {"x-wing": XWing(), "x25519mlkem768": Hybrid("X25519MLKEM768", 0),
            "kyber768-x25519": Hybrid("Kyber768-X25519", 1), "kyber512-x25519": Hybrid("Kyber512-X25519", 2)}


def ByName(name: str):
    """kem/schemes/schemes.go:70 -- case-insensitive lookup; None if unknown."""
    return _SCHEMES.get(name.lower())


def All():
    return list(_SCHEMES.values())
