"""A Python model of P-384 and P-521 and of HPKE's DHKEM over them (RFC 9180 section 4.1, hpke/shortkem.go and
hpke/kembase.go), for the tests: curve constants, affine arithmetic on Python integers, and the labeled KDF on
hashlib / hmac.  `dhkem` runs its ECDH through OpenSSL (cryptography's derive_private_key and ECDH), so it shares no
arithmetic with the device code or with the C oracle.
"""
import hashlib
import hmac
from dataclasses import dataclass


@dataclass(frozen=True)
class Curve:
    name: str
    kem_id: int
    bits: int
    p: int
    n: int
    b: int
    g: tuple
    hash: object  # hashlib constructor of the KDF
    mask0: int  # DeriveKeyPair's bitmask on the candidate's first byte

    @property
    def nbytes(self):
        return (self.bits + 7) // 8

    @property
    def npk(self):
        return 1 + 2 * self.nbytes

    @property
    def nss(self):
        return self.hash().digest_size

    def ossl(self):
        from cryptography.hazmat.primitives.asymmetric import ec
        return ec.SECP384R1() if self.bits == 384 else ec.SECP521R1()


P384 = Curve(
    "P-384", 0x11, 384, 2**384 - 2**128 - 2**96 + 2**32 - 1,
    0xffffffffffffffffffffffffffffffffffffffffffffffffc7634d81f4372ddf581a0db248b0a77aecec196accc52973,
    0xb3312fa7e23ee7e4988e056be3f82d19181d9c6efe8141120314088f5013875ac656398d8a2ed19d2a85c8edd3ec2aef,
    (0xaa87ca22be8b05378eb1c71ef320ad746e1d3b628ba79b9859f741e082542a385502f25dbf55296c3a545e3872760ab7,
     0x3617de4a96262c6f5d9e98bf9292dc29f8f41dbd289a147ce9da3113b5f0b8c00a60b1ce1d7e819d7a431d7c90ea0e5f),
    hashlib.sha384, 0xff)
P521 = Curve(
    "P-521", 0x12, 521, 2**521 - 1,
    0x01fffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffa51868783bf2f966b7fcc0148f709a5d03bb5c9b8899c47aebb6fb71e91386409,
    0x0051953eb9618e1c9a1f929a21a0b68540eea2da725b99b315f3b8b489918ef109e156193951ec7e937b1652c0bd3bb1bf073573df883d2c34f1ef451fd46b503f00,
    (0x00c6858e06b70404e9cd9e3ecb662395b4429c648139053fb521f828af606b4d3dbaa14b5e77efe75928fe1dc127a2ffa8de3348b3c1856a429bf97e7e31c2e5bd66,
     0x011839296a789a3bc0045c8a5fb42c7d1bd998f54449579b446817afbd17273e662c97ee72995ef42640c550b9013fad0761353c7086a272c24088be94769fd16650),
    hashlib.sha512, 0x01)
CURVES = {384: P384, 521: P521}


# ---------------------------------------------------------------- affine arithmetic (None = the point at infinity)
def add(c: Curve, a, b):
    if a is None:
        return b
    if b is None:
        return a
    P = c.p
    if a[0] == b[0]:
        if (a[1] + b[1]) % P == 0:
            return None
        lam = (3 * a[0] * a[0] - 3) * pow(2 * a[1], -1, P) % P
    else:
        lam = (b[1] - a[1]) * pow(b[0] - a[0], -1, P) % P
    x = (lam * lam - a[0] - b[0]) % P
    return x, (lam * (a[0] - x) - a[1]) % P


def mul(c: Curve, k, pt):
    r = None
    for bit in bin(k)[2:]:
        r = add(c, r, r)
        if bit == "1":
            r = add(c, r, pt)
    return r


def enc(c: Curve, pt) -> bytes:
    return b"\x04" + pt[0].to_bytes(c.nbytes, "big") + pt[1].to_bytes(c.nbytes, "big")


def point_ok(c: Curve, b: bytes) -> bool:
    if len(b) != c.npk or b[0] != 4:
        return False
    x, y = int.from_bytes(b[1:1 + c.nbytes], "big"), int.from_bytes(b[1 + c.nbytes:], "big")
    return x < c.p and y < c.p and (y * y - (x * x * x - 3 * x + c.b)) % c.p == 0


def scalar_ok(c: Curve, b: bytes) -> bool:
    return 0 < int.from_bytes(b, "big") < c.n


# ---------------------------------------------------------------- the labeled KDF (RFC 9180 section 4)
def labeled_extract(c: Curve, salt: bytes, label: bytes, ikm: bytes) -> bytes:
    sid = b"KEM" + c.kem_id.to_bytes(2, "big")
    return hmac.new(salt or bytes(c.nss), b"HPKE-v1" + sid + label + ikm, c.hash).digest()


def labeled_expand(c: Curve, prk: bytes, label: bytes, info: bytes, L: int) -> bytes:
    """HKDF-Expand over as many blocks as L needs."""
    sid = b"KEM" + c.kem_id.to_bytes(2, "big")
    linfo = L.to_bytes(2, "big") + b"HPKE-v1" + sid + label + info
    out, t, i = b"", b"", 1
    while len(out) < L:
        t = hmac.new(prk, t + linfo + bytes([i]), c.hash).digest()
        out, i = out + t, i + 1
    return out[:L]


# ---------------------------------------------------------------- DHKEM, with OpenSSL's ECDH
def _ossl_pub(c: Curve, sk: bytes) -> bytes:
    from cryptography.hazmat.primitives import serialization as ser
    from cryptography.hazmat.primitives.asymmetric import ec
    k = ec.derive_private_key(int.from_bytes(sk, "big"), c.ossl())
    return k.public_key().public_bytes(ser.Encoding.X962, ser.PublicFormat.UncompressedPoint)


def _ossl_dh(c: Curve, sk: bytes, pk: bytes) -> bytes:
    from cryptography.hazmat.primitives.asymmetric import ec
    k = ec.derive_private_key(int.from_bytes(sk, "big"), c.ossl())
    return k.exchange(ec.ECDH(), ec.EllipticCurvePublicKey.from_encoded_point(c.ossl(), pk))


def derive_key_pair(c: Curve, seed: bytes):
    """shortkem.go:63-90: (pk, sk)."""
    prk = labeled_extract(c, b"", b"dkp_prk", seed)
    for ctr in range(256):
        sk = bytearray(labeled_expand(c, prk, b"candidate", bytes([ctr]), c.nbytes))
        sk[0] &= c.mask0
        if scalar_ok(c, bytes(sk)):
            return _ossl_pub(c, bytes(sk)), bytes(sk)
    raise AssertionError("no candidate")


def _kdf(c: Curve, dh: bytes, ctx: bytes) -> bytes:
    return labeled_expand(c, labeled_extract(c, b"", b"eae_prk", dh), b"shared_secret", ctx, c.nss)


def encaps(c: Curve, pkR: bytes, seed: bytes, skS: bytes = None):
    """(enc, ss): Encap, or AuthEncap with skS (kembase.go:120-183); valid keys only."""
    enc_, skE = derive_key_pair(c, seed)
    dh, ctx = _ossl_dh(c, skE, pkR), enc_ + pkR
    if skS is not None:
        dh, ctx = dh + _ossl_dh(c, skS, pkR), ctx + _ossl_pub(c, skS)
    return enc_, _kdf(c, dh, ctx)


def decaps(c: Curve, skR: bytes, enc_: bytes, pkS: bytes = None) -> bytes:
    dh, ctx = _ossl_dh(c, skR, enc_), enc_ + _ossl_pub(c, skR)
    if pkS is not None:
        dh, ctx = dh + _ossl_dh(c, skR, pkS), ctx + pkS
    return _kdf(c, dh, ctx)


# ---------------------------------------------------------------- RFC 9180 section 5.1, base mode
def schedule(c: Curve, ss: bytes, info: bytes):
    """(AESGCM(key), base_nonce) of the suite (this KEM, its own HKDF, AES-256-GCM) for a KEM shared secret ss."""
    from cryptography.hazmat.primitives.ciphers.aead import AESGCM
    kdf = 0x0002 if c.bits == 384 else 0x0003
    sid = b"HPKE" + c.kem_id.to_bytes(2, "big") + kdf.to_bytes(2, "big") + (2).to_bytes(2, "big")
    nh = c.nss
    ext = lambda salt, lab, ikm: hmac.new(salt or bytes(nh), b"HPKE-v1" + sid + lab + ikm, c.hash).digest()  # noqa: E731
    exp = lambda prk, lab, inf, L: hmac.new(prk, L.to_bytes(2, "big") + b"HPKE-v1" + sid + lab + inf + b"\x01",  # noqa: E731
                                            c.hash).digest()[:L]
    ctx = b"\x00" + ext(b"", b"psk_id_hash", b"") + ext(b"", b"info_hash", info)
    secret = ext(ss, b"secret", b"")
    return AESGCM(exp(secret, b"key", ctx, 32)), exp(secret, b"base_nonce", ctx, 12)
