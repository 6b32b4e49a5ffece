"""RSA blind signatures (RFC 9474, RSABSSA-SHA384) over the C ABI, server side: the reference's blindsign/blindrsa
package (brsa.go) for its four variants.  The client side (Prepare, Blind, Finalize) is not served here.

  SHA384PSSRandomized, SHA384PSSZeroRandomized, SHA384PSSDeterministic, SHA384PSSZeroDeterministic   Variant (ids 0-3)
  NewSigner(sk).BlindSign(data)                    brsa.go:237-257, with DecryptAndCheck's check s^e mod N == c
  NewVerifier(variant, pk).Verify(message, sig)    brsa.go:202-216
  .BlindSignBatch / .VerifyBatch                   the same on batches (numpy arrays or CUDA tensors)

Keys are plain classes: PrivateKey(N, E, D, Primes) and PublicKey(N, E) with Python integers, as in crypto/rsa.  The
signer derives dp = D mod (p - 1), dq = D mod (q - 1) and qinv = q^-1 mod p as PrivateKey.Precompute does.  Served keys
have two primes of at most 2048 bits each, a modulus of 2048 to 4096 bits and an odd E with 3 <= E < 2^32; NewSigner and
NewVerifier raise ErrInvalidKey for any other, without needing a device.  Other argument errors of a batch call (mixed
host and device buffers, a misaligned device msg_off) raise the library's Cb200Error.

A batch whose ops fail raises the error of the first failure class, with .status holding the per-op bytes and .results
the outputs, whose failed rows are all zero.  BlindSign: 1 = c > N (ErrInvalidMessageLength), 2 = the check failed
(ErrInternal, the reference's "rsa: internal error").  Verify: 1 = s >= N, 2 = an inconsistent EMSA-PSS encoding (both
ErrVerification, as in the reference).
"""
from __future__ import annotations

import numpy as np

from ._ffi import check, lib
from .hybrid import _is_torch, _new, _prep, _ptr

__all__ = ["SHA384PSSRandomized", "SHA384PSSZeroRandomized", "SHA384PSSDeterministic", "SHA384PSSZeroDeterministic",
           "PrivateKey", "PublicKey", "NewSigner", "NewVerifier", "Signer", "Verifier", "BlindRSAError",
           "ErrInvalidVariant", "ErrUnexpectedSize", "ErrInvalidMessageLength", "ErrInternal", "ErrVerification",
           "ErrInvalidKey"]

SHA384PSSRandomized, SHA384PSSZeroRandomized, SHA384PSSDeterministic, SHA384PSSZeroDeterministic = 0, 1, 2, 3
_NAMES = ["RSABSSA-SHA384-PSS-Randomized", "RSABSSA-SHA384-PSSZERO-Randomized", "RSABSSA-SHA384-PSS-Deterministic",
          "RSABSSA-SHA384-PSSZERO-Deterministic"]


class BlindRSAError(ValueError):
    def __init__(self, msg="", status=None, results=None):
        super().__init__(msg)
        self.status, self.results = status, results


class ErrInvalidVariant(BlindRSAError):  # common.ErrInvalidVariant
    pass


class ErrUnexpectedSize(BlindRSAError):  # common.ErrUnexpectedSize: a row that is not kLen bytes
    pass


class ErrInvalidMessageLength(BlindRSAError):  # common.ErrInvalidMessageLength: c > N
    pass


class ErrInternal(BlindRSAError):  # DecryptAndCheck's "rsa: internal error": s^e mod N != c
    pass


class ErrVerification(BlindRSAError):  # rsa.ErrVerification
    pass


class ErrInvalidKey(BlindRSAError):  # a key outside the served range (CB200_ERR_ARG)
    pass


class PublicKey:
    def __init__(self, N: int, E: int):
        self.N, self.E = int(N), int(E)

    def Size(self) -> int:
        return (self.N.bit_length() + 7) // 8


class PrivateKey:
    def __init__(self, N: int, E: int, D: int, Primes):
        self.N, self.E, self.D, self.Primes = int(N), int(E), int(D), [int(p) for p in Primes]
        self.PublicKey = PublicKey(N, E)


def _be(x: int) -> bytes:
    return x.to_bytes((x.bit_length() + 7) // 8 or 1, "big")


def _check_key(rc):
    """the rc of a call with n = 0, which checks the key (and nothing the batch holds) without needing a device"""
    if rc == -1:
        raise ErrInvalidKey(lib().cb200_last_error().decode())


def _rows(x, klen):
    if isinstance(x, (bytes, bytearray)):
        x = np.frombuffer(bytes(x), dtype=np.uint8).reshape(1, -1)
    return _prep(x, klen, ErrUnexpectedSize(f"blindrsa: rows must be (n, {klen}) uint8"))


def _strings(x):
    """(bytes, offsets, n) of a list of bytes (host arrays) or of (bytes, offsets) CUDA tensors"""
    if isinstance(x, tuple) and _is_torch(x[0]):
        data, off = x
        return data, off, off.shape[0] - 1
    lens = [len(m) for m in x]
    off = np.zeros(len(x) + 1, dtype=np.uint64)
    np.cumsum(lens, out=off[1:])
    data = np.frombuffer(b"".join(bytes(m) for m in x) or b"\0", dtype=np.uint8).copy()
    return data, off, len(x)


def _host(st):
    return st.cpu().numpy() if _is_torch(st) else st


def _raise_sign_status(st, sig, n, scheme):
    """raises the error of the first failing BlindSign status class (1, then 2) of a batch, if any"""
    s = _host(st)
    for bit, cls, what in ((1, ErrInvalidMessageLength, "invalid message length"), (2, ErrInternal, "internal error")):
        if (s == bit).any():
            raise cls(f"{scheme}: {what} in {int((s == bit).sum())} of {n} ops", st, sig)


class Signer:
    """Signer of brsa.go: BlindSign under one private key."""

    def __init__(self, sk: PrivateKey):
        if len(sk.Primes) != 2:
            raise ErrInvalidKey("blindrsa: only two-prime keys are served")
        p, q = sk.Primes
        self.sk = sk
        self._fields = [_be(v) for v in (sk.N, sk.E, p, q, sk.D % (p - 1), sk.D % (q - 1), pow(q, -1, p))]
        self.kLen = sk.PublicKey.Size()
        z = np.zeros(1, np.uint8)
        _check_key(lib().cb200_brsa_blind_sign(*self._args(), z.ctypes.data, z.ctypes.data, z.ctypes.data, 0))

    def _args(self):
        args = []
        for f in self._fields:
            args += [f, len(f)]
        return args

    def BlindSignBatch(self, blinded):
        """blind signatures (n, kLen) of blinded messages (n, kLen)"""
        data = _rows(blinded, self.kLen)
        n = data.shape[0]
        sig, st = _new(data, (n, self.kLen)), _new(data, (n,))
        check(lib().cb200_brsa_blind_sign(*self._args(), _ptr(data), _ptr(sig), _ptr(st), n))
        _raise_sign_status(st, sig, n, "blindrsa")
        return sig

    def BlindSign(self, data: bytes) -> bytes:
        """brsa.go:237-257"""
        if len(data) != self.kLen:
            raise ErrUnexpectedSize("blindrsa: unexpected input size")
        return _host(self.BlindSignBatch(bytes(data)))[0].tobytes()


class Verifier:
    """Verifier of brsa.go: Verify under one public key and variant."""

    def __init__(self, variant: int, pk: PublicKey):
        if variant not in (0, 1, 2, 3):
            raise ErrInvalidVariant("blindrsa: invalid BRSA variant")
        self.variant, self.pk = variant, pk
        self._n, self._e = _be(pk.N), _be(pk.E)
        self.kLen = pk.Size()
        z, off = np.zeros(1, np.uint8), np.zeros(1, np.uint64)
        _check_key(lib().cb200_brsa_verify(variant, self._n, len(self._n), self._e, len(self._e), z.ctypes.data,
                                           off.ctypes.data, z.ctypes.data, z.ctypes.data, 0))

    def __repr__(self):
        return _NAMES[self.variant]

    def VerifyBatch(self, messages, sigs):
        """status bytes (n,) of messages (a list of bytes, or (msgs, msg_off) CUDA tensors: uint8 bytes and n + 1
        int64 offsets) and signatures (n, kLen); raises ErrVerification if any op fails"""
        msgs, off, n = _strings(messages)
        sig = _rows(sigs, self.kLen)
        if sig.shape[0] != n:
            raise ErrUnexpectedSize("blindrsa: one signature per message")
        st = _new(sig, (n,))
        if n:
            check(lib().cb200_brsa_verify(self.variant, self._n, len(self._n), self._e, len(self._e), _ptr(msgs),
                                          _ptr(off), _ptr(sig), _ptr(st), n))
        s = _host(st)
        if s.any():
            raise ErrVerification(f"blindrsa: verification error in {int((s != 0).sum())} of {n} ops", st, None)
        return st

    def Verify(self, message: bytes, signature: bytes) -> None:
        """brsa.go:214; raises ErrVerification"""
        if len(signature) != self.kLen:
            raise ErrVerification("crypto/rsa: verification error")
        self.VerifyBatch([bytes(message)], bytes(signature))


def NewSigner(sk: PrivateKey) -> Signer:
    return Signer(sk)


def NewVerifier(variant: int, pk: PublicKey) -> Verifier:
    return Verifier(variant, pk)
