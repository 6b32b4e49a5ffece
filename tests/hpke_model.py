"""An independent model of the two HPKE DHKEMs (RFC 9180 section 4.1, as the reference's hpke/kembase.go and
hpke/xkem.go compute them), built from OpenSSL's X25519 / X448 and Python's hmac / hashlib.

A failed DH (a low-order peer key, where the reference's Shared returns false) raises LowOrder, which stands for
hpke.ErrInvalidKEMSharedSecret.  OpenSSL refuses those points on its own (an all-zero result), so they are recognised
here by that refusal.
"""
from __future__ import annotations

import hashlib
import hmac

from cryptography.hazmat.primitives.asymmetric import x448, x25519

X25519_ID, X448_ID = 0x20, 0x21


class LowOrder(Exception):
    pass


class _Kem:
    def __init__(self, kem_id, h, n, priv, pub):
        self.id, self.h, self.n, self._priv, self._pub = kem_id, h, n, priv, pub
        self.nh = h().digest_size
        self.suite = b"KEM" + kem_id.to_bytes(2, "big")

    def extract(self, salt: bytes, label: bytes, ikm: bytes) -> bytes:
        return hmac.new(salt or bytes(self.nh), b"HPKE-v1" + self.suite + label + ikm, self.h).digest()

    def expand(self, prk: bytes, label: bytes, info: bytes, L: int) -> bytes:
        info = L.to_bytes(2, "big") + b"HPKE-v1" + self.suite + label + info
        out, t, i = b"", b"", 1
        while len(out) < L:
            t = hmac.new(prk, t + info + bytes([i]), self.h).digest()
            out, i = out + t, i + 1
        return out[:L]

    def derive(self, seed: bytes):
        """(sk, pk): DeriveKeyPair; sk unclamped."""
        sk = self.expand(self.extract(b"", b"dkp_prk", seed), b"sk", b"", self.n)
        return sk, self.pub(sk)

    def pub(self, sk: bytes) -> bytes:
        return self._priv.from_private_bytes(sk).public_key().public_bytes_raw()

    def shared(self, sk: bytes, pk: bytes) -> bytes:
        try:
            return self._priv.from_private_bytes(sk).exchange(self._pub.from_public_bytes(pk))
        except ValueError:
            raise LowOrder from None

    def kdf(self, dh: bytes, ctx: bytes) -> bytes:
        return self.expand(self.extract(b"", b"eae_prk", dh), b"shared_secret", ctx, self.nh)

    def encaps(self, pkR: bytes, seed: bytes):
        skE, enc = self.derive(seed)
        return enc, self.kdf(self.shared(skE, pkR), enc + pkR)

    def decaps(self, skR: bytes, enc: bytes) -> bytes:
        return self.kdf(self.shared(skR, enc), enc + self.pub(skR))

    def auth_encaps(self, pkR: bytes, skS: bytes, seed: bytes):
        skE, enc = self.derive(seed)
        dh = self.shared(skE, pkR) + self.shared(skS, pkR)
        return enc, self.kdf(dh, enc + pkR + self.pub(skS))

    def auth_decaps(self, skR: bytes, enc: bytes, pkS: bytes) -> bytes:
        dh = self.shared(skR, enc) + self.shared(skR, pkS)
        return self.kdf(dh, enc + self.pub(skR) + pkS)


KEMS = {X25519_ID: _Kem(X25519_ID, hashlib.sha256, 32, x25519.X25519PrivateKey, x25519.X25519PublicKey),
        X448_ID: _Kem(X448_ID, hashlib.sha512, 56, x448.X448PrivateKey, x448.X448PublicKey)}

# u-coordinates that fail the reference's Shared: X25519's small-order list (dh/x25519/curve.go:89-125, with and
# without bit 255) and X448's residues 0, 1 and p - 1 (dh/x448/curve.go:76-104)
_P25519, _P448 = 2**255 - 19, 2**448 - 2**224 - 1
_X25519_LOW = [0, 1, 325606250916557431795983626356110631294008115727848805560023387167927233504,
               39382357235489614581723060781553021112529911719440698176882885853963445705823,
               _P25519 - 1, _P25519, _P25519 + 1]


def low_order_points(kem_id: int):
    if kem_id == X25519_ID:
        base = [u.to_bytes(32, "little") for u in _X25519_LOW]
        return base + [b[:31] + bytes([b[31] | 0x80]) for b in base]
    return [u.to_bytes(56, "little") for u in (0, 1, _P448 - 1)]
