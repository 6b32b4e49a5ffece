"""Partially blind RSA signatures (draft-amjad-cfrg-partially-blind-rsa, RSAPBSSA-SHA384) over the C ABI, server side:
the reference's blindsign/blindrsa/partiallyblindrsa package (pbrsa.go).  Every op carries public metadata (an expiry,
a policy) that selects the key it is signed and verified under.  The client side (Blind, FixedBlind, Finalize) is not
served here.

  NewSigner(sk, SHA384).BlindSign(data, metadata)            pbrsa.go:350-375
  NewVerifier(pk, SHA384).Verify(message, metadata, sig)     pbrsa.go:244-251
  .BlindSignBatch / .VerifyBatch                             the same on batches, one metadata string per op

Keys are blindrsa's PrivateKey(N, E, D, Primes) and PublicKey(N, E); E and D are not used.  The signer computes
qinv = q^-1 mod p itself.  NewSigner runs NewSigner's safe-prime test once (20 Miller-Rabin rounds on (p - 1) / 2 and
(q - 1) / 2, on the host) and raises ErrInvalidPrivateKey for a key that fails it or lies outside the served range
(two primes = 3 mod 4 of at most 2048 bits each, a modulus of 2048 to 4096 bits); NewVerifier raises
ErrInvalidPublicKey for a modulus outside the range.  Only SHA-384 is served: any other hash is a ValueError, raised
before the library is called.

Batches take blinded messages or signatures as (n, kLen) numpy arrays or CUDA tensors, and messages and metadata as
lists of bytes, or as (bytes, offsets) CUDA tensors: uint8 bytes and n + 1 int64 offsets.  A batch whose ops fail
raises the error of the first failure class, with .status holding the per-op bytes and .results the outputs, whose
failed rows are all zero.  BlindSign: 1 = c > N (ErrInvalidMessageLength), 2 = the check s^e' mod N == c failed
(ErrInternal).  Verify: 1 = s >= N, 2 = an inconsistent EMSA-PSS encoding (both ErrVerification).
"""
from __future__ import annotations

import numpy as np

from ._ffi import check, lib
from .blindrsa import (BlindRSAError, ErrInternal, ErrInvalidMessageLength, ErrUnexpectedSize, ErrVerification,
                       PrivateKey, PublicKey, _be, _host, _raise_sign_status, _rows, _strings)
from .hybrid import _new, _ptr

__all__ = ["SHA384", "NewSigner", "NewVerifier", "Signer", "Verifier", "PrivateKey", "PublicKey",
           "ErrInvalidPrivateKey", "ErrInvalidPublicKey", "ErrUnexpectedSize", "ErrInvalidMessageLength", "ErrInternal",
           "ErrVerification"]

SHA384 = "SHA384"  # crypto.SHA384, the one hash served


class ErrInvalidPrivateKey(BlindRSAError):  # partiallyblindrsa.ErrInvalidPrivateKey
    pass


class ErrInvalidPublicKey(BlindRSAError):  # partiallyblindrsa.ErrInvalidPublicKey
    pass


def _check_hash(h):
    if h != SHA384:
        raise ValueError("partiallyblindrsa: only SHA384 is served")


class Signer:
    """Signer of pbrsa.go: BlindSign under one private key, each op under the key of its metadata."""

    def __init__(self, sk: PrivateKey, hash=SHA384):
        _check_hash(hash)
        if len(sk.Primes) != 2:
            raise ErrInvalidPrivateKey("partiallyblindrsa: only two-prime keys are served")
        p, q = sk.Primes
        self.sk = sk
        self._n, self._p, self._q = _be(sk.N), _be(p), _be(q)
        try:
            qinv = pow(q, -1, p)
        except ValueError:  # not coprime: the library refuses the key
            qinv = 0
        self._qinv = _be(qinv)
        self.kLen = sk.PublicKey.Size()
        z, off = np.zeros(1, np.uint8), np.zeros(1, np.uint64)
        if lib().cb200_pbrsa_blind_sign(*self._key(), z.ctypes.data, z.ctypes.data, off.ctypes.data, z.ctypes.data,
                                        z.ctypes.data, 0) == -1 or \
                lib().cb200_pbrsa_check_key(self._n, len(self._n), self._p, len(self._p), self._q, len(self._q)) == -1:
            raise ErrInvalidPrivateKey(lib().cb200_last_error().decode())

    def _key(self):
        return [self._n, len(self._n), self._p, len(self._p), self._q, len(self._q), self._qinv, len(self._qinv)]

    def BlindSignBatch(self, blinded, metadata):
        """blind signatures (n, kLen) of blinded messages (n, kLen), op i under metadata[i]"""
        data = _rows(blinded, self.kLen)
        n = data.shape[0]
        meta, off, nm = _strings(metadata)
        if nm != n:
            raise ErrUnexpectedSize("partiallyblindrsa: one metadata string per blinded message")
        sig, st = _new(data, (n, self.kLen)), _new(data, (n,))
        if n:
            check(lib().cb200_pbrsa_blind_sign(*self._key(), _ptr(data), _ptr(meta), _ptr(off), _ptr(sig), _ptr(st),
                                               n))
        _raise_sign_status(st, sig, n, "partiallyblindrsa")
        return sig

    def BlindSign(self, data: bytes, metadata: bytes) -> bytes:
        """pbrsa.go:350-375"""
        if len(data) != self.kLen:
            raise ErrUnexpectedSize("partiallyblindrsa: unexpected input size")
        return _host(self.BlindSignBatch(bytes(data), [bytes(metadata)]))[0].tobytes()


class Verifier:
    """Verifier of pbrsa.go: Verify under one public key, each op under the key of its metadata."""

    def __init__(self, pk: PublicKey, hash=SHA384):
        _check_hash(hash)
        self.pk = pk
        self._n = _be(pk.N)
        self.kLen = pk.Size()
        z, off = np.zeros(1, np.uint8), np.zeros(1, np.uint64)
        if lib().cb200_pbrsa_verify(self._n, len(self._n), z.ctypes.data, off.ctypes.data, z.ctypes.data,
                                    off.ctypes.data, z.ctypes.data, z.ctypes.data, 0) == -1:
            raise ErrInvalidPublicKey(lib().cb200_last_error().decode())

    def VerifyBatch(self, messages, metadata, sigs):
        """status bytes (n,) of messages, metadata and signatures (n, kLen); raises ErrVerification if any op fails"""
        msgs, moff, n = _strings(messages)
        meta, off, nm = _strings(metadata)
        sig = _rows(sigs, self.kLen)
        if sig.shape[0] != n or nm != n:
            raise ErrUnexpectedSize("partiallyblindrsa: one signature and one metadata string per message")
        st = _new(sig, (n,))
        if n:
            check(lib().cb200_pbrsa_verify(self._n, len(self._n), _ptr(msgs), _ptr(moff), _ptr(meta), _ptr(off),
                                           _ptr(sig), _ptr(st), n))
        s = _host(st)
        if s.any():
            raise ErrVerification(f"partiallyblindrsa: verification error in {int((s != 0).sum())} of {n} ops", st,
                                  None)
        return st

    def Verify(self, message: bytes, metadata: bytes, signature: bytes) -> None:
        """pbrsa.go:244-251; raises ErrVerification"""
        if len(signature) != self.kLen:
            raise ErrVerification("crypto/rsa: verification error")
        self.VerifyBatch([bytes(message)], [bytes(metadata)], bytes(signature))


def NewSigner(sk: PrivateKey, hash=SHA384) -> Signer:
    return Signer(sk, hash)


def NewVerifier(pk: PublicKey, hash=SHA384) -> Verifier:
    return Verifier(pk, hash)
