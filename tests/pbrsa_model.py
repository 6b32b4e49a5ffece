"""Partially blind RSA (RSAPBSSA-SHA384) restated in pure Python, server and client, for the tests: the reference's
blindsign/blindrsa/partiallyblindrsa package (pbrsa.go).  hashlib and hmac only; the PSS helpers are brsa_model's.

  key        derive_public_key (e' of the metadata), derive_private (d' = e'^-1 mod phi(N))
  server     blind_sign and verify_status, with the status bytes of the C ABI
  client     blind (EMSA-PSS-ENCODE of the framed message, then m r^e' mod N) and finalize
  keys       tests/golden/pbrsa_keys.json.gz
"""
import gzip
import hashlib
import hmac
import json
import os

import brsa_model as bm

HLEN = 48
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def hkdf(salt, ikm, info, length):
    """HKDF-SHA-384 (RFC 5869)"""
    prk = hmac.new(salt, ikm, hashlib.sha384).digest()
    out, t, i = b"", b"", 1
    while len(out) < length:
        t = hmac.new(prk, t + info + bytes([i]), hashlib.sha384).digest()
        out, i = out + t, i + 1
    return out[:length]


def derive_public_key(n, metadata):
    """e' of derivePublicKey (pbrsa.go:81-117)"""
    lam = n.bit_length() // 2
    klen = (n.bit_length() + 7) // 8
    raw = hkdf(n.to_bytes(klen, "big"), b"key" + metadata + b"\x00", b"PBRSA", (lam + 128) // 8)
    e = int.from_bytes(raw[:lam // 8], "big") | 1
    return e & ~(1 << (lam - 1)) & ~(1 << (lam - 2))


def derive_private(k, metadata):
    """(e', d') of deriveKeyPair (pbrsa.go:123-144)"""
    e = derive_public_key(k.n, metadata)
    return e, pow(e, -1, (k.p - 1) * (k.q - 1))


def frame(message, metadata):
    """encodeMessageMetadata (pbrsa.go:22-28)"""
    return b"msg" + len(metadata).to_bytes(4, "big") + metadata + message


# ---------------------------------------------------------------- server, with the status bytes of the C ABI
def blind_sign(k, blinded, metadata, qinv=None):
    """(status, blind signature): 1 for c > N, 2 for a failed s^e' mod N == c check (then an all-zero row).  With qinv
    given, the CRT route of the library under that (possibly wrong) qinv."""
    c = bm.os2ip(blinded)
    if c > k.n:
        return 1, bytes(k.klen)
    e, d = derive_private(k, metadata)
    if qinv is None:
        s = pow(c, d, k.n)
    else:
        sp, sq = pow(c, d % (k.p - 1), k.p), pow(c, d % (k.q - 1), k.q)
        s = sq + k.q * ((sp - sq) * qinv % k.p)
    if pow(s, e, k.n) != c:
        return 2, bytes(k.klen)
    return 0, bm.i2osp(s, k.klen)


def verify_status(k, message, metadata, sig):
    """0, 1 for s >= N, 2 for an inconsistent encoding"""
    pk = bm.Key(k.n, derive_public_key(k.n, metadata))
    return bm.verify_status(pk, HLEN, frame(message, metadata), sig)


# ---------------------------------------------------------------- client
def blind(k, message, metadata, salt, r):
    """(blinded message, inv = r^-1 mod N) with the given salt and r"""
    e = derive_public_key(k.n, metadata)
    embits = k.n.bit_length() - 1
    m = bm.os2ip(bm.emsa_pss_encode(frame(message, metadata), embits, salt))
    return bm.i2osp(m * pow(r, e, k.n) % k.n, k.klen), pow(r, -1, k.n)


def finalize(k, message, metadata, blind_sig, inv):
    sig = bm.i2osp(bm.os2ip(blind_sig) * inv % k.n, k.klen)
    assert verify_status(k, message, metadata, sig) == 0
    return sig


def sign(k, message, metadata, rng):
    """a final signature: blind, sign, finalize with the model"""
    salt = rng.randbytes(HLEN)
    r = rng.randrange(2, k.n - 1)
    blinded, inv = blind(k, message, metadata, salt, r)
    st, bs = blind_sign(k, blinded, metadata)
    assert st == 0
    return finalize(k, message, metadata, bs, inv)


# ---------------------------------------------------------------- fixtures
def keys():
    """every fixture key by name: strong2048 (the reference's), safe3072, safe4096, safe2050, safe2052, safe3073,
    safe2048u"""
    with gzip.open(os.path.join(GOLDEN, "pbrsa_keys.json.gz")) as f:
        ks = json.load(f)
    return {name: bm.Key(*(int(v[x], 16) for x in ("n", "e", "d", "p", "q"))) for name, v in ks.items()}
