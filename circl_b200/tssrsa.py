"""Threshold RSA signatures over the C ABI: the reference's tss/rsa package (Shoup's protocol 1, "Practical Threshold
Signatures").  A dealer splits an RSA key into `players` key shares, any `threshold` of which sign together.

  Deal(rand, players, threshold, key, cache)          rsa_threshold.go:95-167 (host, Python integers)
  PadHash(padder, hash, pub, msg)                     with PKCS1v15Padder or PSSPadder (host, hashlib)
  KeyShare.Sign(rand, pub, digest, parallel)          keyshare.go:188-256: xi = x^(2 Delta s_i) mod N on the GPU
  KeyShare.SignBatch(pub, digests)                    the same for a batch of digests (numpy rows or CUDA tensors)
  CombineSignShares(pub, players, threshold, shares, msg)             rsa_threshold.go:207-293 on the GPU
  CombineSignSharesBatch(pub, players, threshold, idx, xi, msgs)      the same for a batch of ops
  KeyShare / SignShare .MarshalBinary / .UnmarshalBinary              byte-compatible with keyshare.go / signShare.go

Served beyond the reference's own checks: N of 2048 to 4096 bits, an odd e with 3 <= e < 2^32, 2 <= players <= 64 (the
reference has no bound) and at most 64 shares per op.  A key share's exponent 2 Delta s_i (or its cached twoDeltaSi) has
at most bitlen(N) - 2 + bitlen(2 Delta) bits, as every dealt share does; the constant-time exponentiation runs over that
bound.  Arguments outside these rules raise the library's Cb200Error.

A batch whose ops fail raises the error of the first failure class, with .status holding the per-op bytes and .results
the signatures, whose failed rows are all zero: 1 = ErrInvalidCalc (an index 0, or a Lagrange coefficient that is not
an integer), 2 = ErrInternal (y^e mod N != x, the reference's "rsa: internal error").
"""
from __future__ import annotations

import hashlib
import math

import numpy as np

from ._ffi import check, lib
from .hybrid import _is_torch, _new, _prep, _ptr

__all__ = ["KeyShare", "SignShare", "Deal", "PadHash", "PKCS1v15Padder", "PSSPadder", "CombineSignShares",
           "CombineSignSharesBatch", "TSSRSAError", "ErrInvalidCalc", "ErrInternal", "MAX_PLAYERS"]

MAX_PLAYERS = 64


class TSSRSAError(ValueError):
    def __init__(self, msg="", status=None, results=None):
        super().__init__(msg)
        self.status, self.results = status, results


class ErrInvalidCalc(TSSRSAError):  # rsa.ErrInvalidCalc
    def __init__(self, msg="tss/rsa: invalid calculation", status=None, results=None):
        super().__init__(msg, status, results)


class ErrInternal(TSSRSAError):  # CombineSignShares' "rsa: internal error": y^e mod N != x
    pass


def _delta(players: int) -> int:
    """util.go:7-12: Delta = players!"""
    return math.factorial(max(players, 0))


def _be(x: int) -> bytes:
    return x.to_bytes((x.bit_length() + 7) // 8 or 1, "big")


def _u16(v: int) -> bytes:
    return int(v).to_bytes(2, "big")


def _klen(pub) -> int:
    return (pub.N.bit_length() + 7) // 8


def _host(st):
    return st.cpu().numpy() if _is_torch(st) else st


class KeyShare:
    """keyshare.go:15-24: the secret share si, the optional cached twoDeltaSi (used as given when present), Index,
    Players and Threshold"""

    def __init__(self, si: int = 0, Index: int = 0, Players: int = 0, Threshold: int = 0, twoDeltaSi=None):
        self.si, self.Index, self.Players, self.Threshold = int(si), int(Index), int(Players), int(Threshold)
        self.twoDeltaSi = None if twoDeltaSi is None else int(twoDeltaSi)

    def MarshalBinary(self) -> bytes:
        """| Players u16 | Threshold u16 | Index u16 | siLen u16 | si | twoDeltaSiNil u8 | twoDeltaSiLen u16 |
        twoDeltaSi |, big-endian (keyshare.go:33-103)"""
        for v, what in ((self.Players, "Players"), (self.Threshold, "Threshold"), (self.Index, "Index")):
            if v > 0xffff:
                raise ValueError(f"rsa_threshold: keyshare marshall: {what} is too big to fit in a uint16")
        tds = b"" if self.twoDeltaSi is None else self.twoDeltaSi.to_bytes((self.twoDeltaSi.bit_length() + 7) // 8,
                                                                            "big")
        if len(tds) > 0x7fff:
            raise ValueError("rsa_threshold: keyshare marshall: twoDeltaSiBytes is too big to fit its length in a "
                             "uint16")
        si = _be(self.si)
        if len(si) > 0x7fff:
            raise ValueError("rsa_threshold: keyshare marshall: siBytes is too big to fit it's length in a uint16")
        return (_u16(self.Players) + _u16(self.Threshold) + _u16(self.Index) + _u16(len(si)) + si
                + bytes([self.twoDeltaSi is not None]) + _u16(len(tds)) + tds)

    def UnmarshalBinary(self, data: bytes) -> None:
        """keyshare.go:105-161; raises ValueError on an invalid encoding"""
        data = bytes(data)
        pre = "rsa_threshold: keyshare unmarshalKeyShareTest failed: "
        if len(data) < 6:
            raise ValueError(pre + "data length was too short for reading Players, Threshold, Index")
        if len(data) - 6 < 2:
            raise ValueError(pre + "data length was too short for reading siLen length")
        si_len = int.from_bytes(data[6:8], "big")
        if si_len == 0:
            raise ValueError(pre + "si is a required field but siLen was 0")
        if len(data) - 8 < si_len:
            raise ValueError(pre + f"data length was too short for reading si, needed: {si_len} found: {len(data) - 8}")
        si = int.from_bytes(data[8:8 + si_len], "big")
        if len(data) - 8 - si_len < 1:
            raise ValueError(pre + "data length was too short for reading twoDeltaSiNil")
        tds = None
        if data[8 + si_len] != 0:
            o = 8 + si_len + 1
            if len(data) - o < 2:
                raise ValueError(pre + "data length was too short for reading twoDeltaSiLen length")
            tl = int.from_bytes(data[o:o + 2], "big")
            if len(data) - o - 2 < tl:
                raise ValueError(pre + f"data length was too short for reading twoDeltaSi, needed: {tl} found: "
                                 f"{len(data) - o - 2}")
            tds = int.from_bytes(data[o + 2:o + 2 + tl], "big")
        self.Players, self.Threshold, self.Index = (int.from_bytes(data[i:i + 2], "big") for i in (0, 2, 4))
        self.si, self.twoDeltaSi = si, tds

    def get2DeltaSi(self, players: int) -> int:
        """keyshare.go:163-176: the cached twoDeltaSi as given, else 2 Delta si (then cached)"""
        if self.twoDeltaSi is None:
            self.twoDeltaSi = 2 * _delta(players) * self.si
        return self.twoDeltaSi

    def SignBatch(self, pub, digests):
        """the signature shares xi (n, kLen) = x^(2 Delta si) mod N of the digests (n, kLen): numpy rows or a CUDA
        tensor (the result is then a CUDA tensor)"""
        kl = _klen(pub)
        data = _prep(digests, kl, ValueError(f"tssrsa: digests must be (n, {kl}) uint8"))
        n = data.shape[0]
        out = _new(data, (n, kl))
        e = _be(self.get2DeltaSi(self.Players))
        nb = _be(pub.N)
        check(lib().cb200_tssrsa_sign_share(nb, len(nb), self.Players, e, len(e), _ptr(data), _ptr(out), n))
        return out

    def Sign(self, rand, pub, digest: bytes, parallel: bool = True) -> "SignShare":
        """keyshare.go:188-256.  rand and parallel are accepted and not used: the exponentiation is constant-time in
        place of the reference's blinding, whose result does not depend on its random value.  (With blinding, the
        reference fails with "rsa_threshold: no mod inverse" when the digest shares a factor with N; this Sign returns
        the share x^(2 Delta si) mod N for it, as the reference does without blinding.)  A digest longer than kLen bytes
        is reduced mod N on the host, which Exp does too."""
        kl = _klen(pub)
        x = int.from_bytes(bytes(digest), "big")
        if len(digest) > kl:
            x %= pub.N
        row = np.frombuffer(x.to_bytes(kl, "big"), np.uint8).reshape(1, kl).copy()
        xi = self.SignBatch(pub, row)[0].tobytes()
        return SignShare(int.from_bytes(xi, "big"), self.Index, self.Players, self.Threshold)

    def __repr__(self):
        return f"(t,n): ({self.Threshold},{self.Players}) index: {self.Index} si: 0x{self.si:x}"


class SignShare:
    """signShare.go:10-17"""

    def __init__(self, xi: int = 0, Index: int = 0, Players: int = 0, Threshold: int = 0):
        self.xi, self.Index, self.Players, self.Threshold = int(xi), int(Index), int(Players), int(Threshold)

    def MarshalBinary(self) -> bytes:
        """| Players u16 | Threshold u16 | Index u16 | xiLen u16 | xi |, big-endian (signShare.go:27-70)"""
        for v, what in ((self.Players, "Players"), (self.Threshold, "Threshold"), (self.Index, "Index")):
            if v > 0xffff:
                raise ValueError(f"rsa_threshold: signshare marshall: {what} is too big to fit in a uint16")
        xi = _be(self.xi)
        if len(xi) > 0x7fff:
            raise ValueError("rsa_threshold: signshare marshall: xiBytes is too big to fit it's length in a uint16")
        return _u16(self.Players) + _u16(self.Threshold) + _u16(self.Index) + _u16(len(xi)) + xi

    def UnmarshalBinary(self, data: bytes) -> None:
        """signShare.go:72-103; raises ValueError on an invalid encoding"""
        data = bytes(data)
        pre = "rsa_threshold: signshare unmarshalKeyShareTest failed: "
        if len(data) < 8:
            raise ValueError(pre + "data length was too short for reading Players, Threshold, Index, and xiLen")
        xl = int.from_bytes(data[6:8], "big")
        if xl == 0:
            raise ValueError(pre + "xi is a required field but xiLen was 0")
        if len(data) - 8 < xl:
            raise ValueError(pre + f"data length was too short for reading xi, needed: {xl} found: {len(data) - 8}")
        self.Players, self.Threshold, self.Index = (int.from_bytes(data[i:i + 2], "big") for i in (0, 2, 4))
        self.xi = int.from_bytes(data[8:8 + xl], "big")

    def __repr__(self):
        return f"(t,n): ({self.Threshold},{self.Players}) index: {self.Index} xi: 0x{self.xi:x}"


def _validate_params(players: int, threshold: int) -> None:
    """rsa_threshold.go:83-93"""
    if players <= 1:
        raise ValueError("rsa_threshold: Players (l) invalid: should be > 1")
    if threshold < 1 or threshold > players:
        raise ValueError(f"rsa_threshold: Threshold (k) invalid: {threshold} < 1 || {threshold} > {players}")


class _GoRand:
    """crypto/rand.Int over a reader with read(n) -> bytes (an io.Reader), as Go restates it"""

    def __init__(self, reader):
        self.r = reader

    def int_below(self, m: int) -> int:
        bl = (m - 1).bit_length()
        if bl == 0:
            return 0
        k, b = (bl + 7) // 8, bl % 8 or 8
        while True:
            buf = bytearray(self.r.read(k))
            if len(buf) != k:
                raise ValueError("rsa_threshold: unable to generate an int within [0, m)")
            buf[0] &= (1 << b) - 1
            v = int.from_bytes(buf, "big")
            if v < m:
                return v


def Deal(rand, players: int, threshold: int, key, cache: bool) -> list:
    """rsa_threshold.go:95-167 on the host: key has .E and .Primes (two primes); rand has read(n) -> bytes.  The
    polynomial's coefficients come from crypto/rand.Int's rejection sampling, so a seeded byte stream gives the
    reference's shares."""
    _validate_params(players, threshold)
    if len(key.Primes) != 2:
        raise ValueError("multiprime rsa keys are unsupported")
    p, q = (int(v) for v in key.Primes)
    m = ((p - 1) * (q - 1)) >> 2
    try:
        d = pow(int(key.E), -1, m)
    except ValueError:
        raise ValueError("rsa_threshold: no ModInverse for e in Z/Zm") from None
    g = _GoRand(rand)
    a = [d] + [g.int_below(m) for _ in range(threshold - 1)]
    shares = []
    for i in range(1, players + 1):
        s = a[-1]
        for c in reversed(a[:-1]):
            s = (s * i % m + c) % m
        ks = KeyShare(s, i, players, threshold)
        if cache:
            ks.get2DeltaSi(players)
        shares.append(ks)
    return shares


# PKCS #1 v1.5 DigestInfo prefixes by hashlib name (internal/pkcs1v15.go)
_PREFIX = {
    "md5": bytes.fromhex("3020300c06082a864886f70d020505000410"),
    "sha1": bytes.fromhex("3021300906052b0e03021a05000414"),
    "sha224": bytes.fromhex("302d300d06096086480165030402040500041c"),
    "sha256": bytes.fromhex("3031300d060960864801650304020105000420"),
    "sha384": bytes.fromhex("3041300d060960864801650304020205000430"),
    "sha512": bytes.fromhex("3051300d060960864801650304020305000440"),
}


class PKCS1v15Padder:
    def Pad(self, pub, hash: str, hashed: bytes) -> bytes:
        """EMSA-PKCS1-v1_5: 0x00 || 0x01 || 0xff.. || 0x00 || DigestInfo prefix || hashed (kLen bytes)"""
        h = hashlib.new(hash)
        if len(hashed) != h.digest_size:
            raise ValueError("threshold_internal: crypto/rsa: input must be hashed message")
        if hash not in _PREFIX:
            raise ValueError("threshold_internal: crypto/rsa: unsupported hash function")
        t = _PREFIX[hash] + bytes(hashed)
        k = _klen(pub)
        if k < len(t) + 11:
            raise ValueError("message too long")
        return b"\x00\x01" + b"\xff" * (k - len(t) - 3) + b"\x00" + t


class PSSPadder:
    """EMSA-PSS with MGF1 of the same hash.  Rand: read(n) -> bytes for the salt; SaltLength None or 0 = the largest
    salt the key allows (PSSSaltLengthAuto), -1 = the hash length.  Every party must sign the same encoding, so one
    party draws the salt and shares it."""

    def __init__(self, Rand=None, SaltLength=None):
        self.Rand, self.SaltLength = Rand, SaltLength

    def Pad(self, pub, hash: str, hashed: bytes) -> bytes:
        hl = hashlib.new(hash).digest_size
        embits = pub.N.bit_length() - 1
        emlen = (embits + 7) // 8
        slen = emlen - 2 - hl if not self.SaltLength else hl if self.SaltLength == -1 else self.SaltLength
        salt = bytes(self.Rand.read(slen)) if slen else b""
        if len(salt) != slen:
            raise ValueError("unexpected EOF")
        if len(hashed) != hl:
            raise ValueError("crypto/rsa: input must be hashed with given hash")
        if emlen < hl + slen + 2:
            raise ValueError("crypto/rsa: key size too small for PSS signature")
        H = hashlib.new(hash, bytes(8) + bytes(hashed) + salt).digest()
        db = bytearray(bytes(emlen - slen - hl - 2) + b"\x01" + salt)
        mask, c = b"", 0
        while len(mask) < len(db):
            mask += hashlib.new(hash, H + c.to_bytes(4, "big")).digest()
            c += 1
        for i in range(len(db)):
            db[i] ^= mask[i]
        db[0] &= 0xff >> (8 * emlen - embits)
        return bytes(db) + H + b"\xbc"


def PadHash(padder, hash: str, pub, msg: bytes) -> bytes:
    """rsa_threshold.go: Pad(Hash(msg)); hash is a hashlib name"""
    return padder.Pad(pub, hash, hashlib.new(hash, bytes(msg)).digest())


def _combine_call(pub, players, threshold, idx, xi, msgs):
    kl = _klen(pub)
    if _is_torch(xi):
        import torch
        n, k = idx.shape
        if not (idx.is_cuda and idx.element_size() == 2 and idx.is_contiguous()):
            raise ValueError("tssrsa: idx must be a contiguous (n, k) 16-bit CUDA tensor")
        xi = xi.reshape(n, k * kl)
        check(lib().cb200_set_stream(torch.cuda.current_stream().cuda_stream))
    else:
        idx = np.asarray(idx)
        if idx.ndim != 2 or idx.dtype.kind not in "iu":
            raise ValueError("tssrsa: idx must be (n, k) integers")
        if idx.size and (int(idx.min()) < 0 or int(idx.max()) > 0xffff):
            raise ValueError("tssrsa: share indices must be in 0 .. 65535")
        idx = np.ascontiguousarray(idx, dtype=np.uint16)
        n, k = idx.shape
        xi = np.ascontiguousarray(xi, dtype=np.uint8).reshape(n, k * kl)
    xi = _prep(xi, k * kl, ValueError(f"tssrsa: xi must be (n, {k}, {kl}) uint8"))
    msgs = _prep(msgs, kl, ValueError(f"tssrsa: msgs must be (n, {kl}) uint8"))
    if xi.shape[0] != n or msgs.shape[0] != n:
        raise ValueError("tssrsa: idx, xi and msgs need one row per op")
    sig, st = _new(msgs, (n, kl)), _new(msgs, (n,))
    nb, eb = _be(pub.N), _be(pub.E)
    check(lib().cb200_tssrsa_combine(nb, len(nb), eb, len(eb), players, threshold, k, _ptr(idx), _ptr(xi),
                                     _ptr(msgs), _ptr(sig), _ptr(st), n))
    return sig, st


def CombineSignSharesBatch(pub, players: int, threshold: int, idx, xi, msgs):
    """signatures (n, kLen) of n ops, op i combining the k shares xi[i] (k rows of kLen bytes) of the indices idx[i]
    (k uint16) for the padded message msgs[i] (kLen bytes): numpy arrays, or CUDA tensors (idx int16 or uint16).  Every
    share is taken to carry (players, threshold); raises ErrInvalidCalc or ErrInternal with .status and .results if any
    op fails."""
    _validate_params(players, threshold)
    sig, st = _combine_call(pub, players, threshold, idx, xi, msgs)
    s, n = _host(st), st.shape[0]
    for code, cls, what in ((1, ErrInvalidCalc, "invalid calculation"), (2, ErrInternal, "internal error")):
        if (s == code).any():
            raise cls(f"tssrsa: {what} in {int((s == code).sum())} of {n} ops", st, sig)
    return sig


def CombineSignShares(pub, players: int, threshold: int, shares, msg: bytes) -> bytes:
    """rsa_threshold.go:207-293: the reference's parameter errors in its order, then the combination on the GPU"""
    _validate_params(players, threshold)
    if len(shares) == 0:
        raise ValueError("rsa_threshold: no shares provided")
    for s in shares:
        if s.Players != players:
            raise ValueError("rsa_threshold: share players did not match protocol players")
        if s.Threshold != threshold:
            raise ValueError("rsa_threshold: share threshold did not match protocol threshold")
    if len(shares) < threshold:
        raise ValueError("rsa_threshold: insufficient shares for the threshold")
    if any(s.Index == 0 for s in shares):  # checkIndices, before any served-range rule
        raise ErrInvalidCalc()
    if any(s.Index > 0xffff for s in shares):
        raise ValueError("tssrsa: share indices above 65535 are not served")
    kl = _klen(pub)
    x = int.from_bytes(bytes(msg), "big")
    # a share longer than kLen bytes is reduced mod N (Exp does); an x that long is >= N and fails the final check as
    # 2^(8 kLen) - 1 does
    x = min(x, (1 << (8 * kl)) - 1)
    xs = [s.xi % pub.N if s.xi >> (8 * kl) else s.xi for s in shares]
    idx = np.array([[s.Index for s in shares]], np.uint16)
    xi = np.frombuffer(b"".join(v.to_bytes(kl, "big") for v in xs), np.uint8).reshape(1, -1).copy()
    m = np.frombuffer(x.to_bytes(kl, "big"), np.uint8).reshape(1, kl).copy()
    sig, st = _combine_call(pub, players, threshold, idx, xi, m)
    if st[0] == 1:
        raise ErrInvalidCalc()
    if st[0] == 2:
        raise ErrInternal("rsa: internal error")
    return sig[0].tobytes()
