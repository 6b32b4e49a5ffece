"""RSA blind signatures (RFC 9474, RSABSSA-SHA384) restated in pure Python, server and client, for the tests: the
reference's blindsign/blindrsa package (brsa.go) with internal/common/{common,rsa,pss}.go.  hashlib only.

  server   blind_sign (pow(c, d, N) and the check s^e mod N == c) and verify, with the status bytes of the C ABI
  client   prepare, blind (EMSA-PSS-ENCODE, then m r^e mod N) and finalize
  keys     the fixtures of tests/golden/: the RFC 9474 key, the RFC 9500 2048-bit PEM key and brsa_keys.json.gz
"""
import base64
import gzip
import hashlib
import json
import os

HLEN = 48
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
# the reference's Variant order: (name, salt length, message prefix length)
VARIANTS = [("RSABSSA-SHA384-PSS-Randomized", 48, 32), ("RSABSSA-SHA384-PSSZERO-Randomized", 0, 32),
            ("RSABSSA-SHA384-PSS-Deterministic", 48, 0), ("RSABSSA-SHA384-PSSZERO-Deterministic", 0, 0)]


class Key:
    def __init__(self, n, e, d=None, p=None, q=None):
        self.n, self.e, self.d, self.p, self.q = n, e, d, p, q

    @property
    def klen(self):
        return (self.n.bit_length() + 7) // 8

    def crt(self):
        """(dp, dq, qinv) as Go's PrivateKey.Precompute derives them"""
        return self.d % (self.p - 1), self.d % (self.q - 1), pow(self.q, -1, self.p)


def i2osp(x, n):
    return x.to_bytes(n, "big")


def os2ip(b):
    return int.from_bytes(b, "big")


def sha384(b):
    return hashlib.sha384(b).digest()


def mgf1(seed, n):
    out = b""
    for c in range((n + HLEN - 1) // HLEN):
        out += sha384(seed + i2osp(c, 4))
    return out[:n]


def emsa_pss_encode(msg, embits, salt):
    emlen = (embits + 7) // 8
    h = sha384(b"\0" * 8 + sha384(msg) + salt)
    db = b"\0" * (emlen - len(salt) - HLEN - 2) + b"\x01" + salt
    masked = bytearray(x ^ y for x, y in zip(db, mgf1(h, emlen - HLEN - 1)))
    masked[0] &= 0xff >> (8 * emlen - embits)
    return bytes(masked) + h + b"\xbc"


def emsa_pss_verify(msg, em, embits, slen):
    emlen = (embits + 7) // 8
    if len(em) != emlen or emlen < HLEN + slen + 2 or em[-1] != 0xbc:
        return False
    bitmask = 0xff >> (8 * emlen - embits)
    if em[0] & ~bitmask & 0xff:
        return False
    h = em[emlen - HLEN - 1:-1]
    db = bytearray(x ^ y for x, y in zip(em[:emlen - HLEN - 1], mgf1(h, emlen - HLEN - 1)))
    db[0] &= bitmask
    ps = emlen - HLEN - slen - 2
    if any(db[:ps]) or db[ps] != 1:
        return False
    salt = bytes(db[len(db) - slen:]) if slen else b""
    return sha384(b"\0" * 8 + sha384(msg) + salt) == h


# ---------------------------------------------------------------- server, with the status bytes of the C ABI
def blind_sign(sk, blinded):
    """(status, blind signature): 1 for c > N, 2 for a failed s^e mod N == c check (then an all-zero row)"""
    c = os2ip(blinded)
    if c > sk.n:
        return 1, bytes(sk.klen)
    dp, dq, qinv = sk.crt()
    return blind_sign_crt(sk, dp, dq, qinv, blinded)


def blind_sign_crt(sk, dp, dq, qinv, blinded):
    """BlindSign with the CRT fields as given (a wrong one makes the check fail)"""
    c = os2ip(blinded)
    if c > sk.n:
        return 1, bytes(sk.klen)
    sp, sq = pow(c, dp, sk.p), pow(c, dq, sk.q)
    s = sq + sk.q * ((sp - sq) * qinv % sk.p)
    if pow(s, sk.e, sk.n) != c:
        return 2, bytes(sk.klen)
    return 0, i2osp(s, sk.klen)


def verify_status(pk, slen, msg, sig):
    """0, 1 for s >= N, 2 for an inconsistent encoding"""
    s = os2ip(sig)
    if len(sig) != pk.klen or s >= pk.n:
        return 1
    m = pow(s, pk.e, pk.n)
    embits = pk.n.bit_length() - 1
    emlen = (embits + 7) // 8
    if m.bit_length() > 8 * emlen:
        return 2
    return 0 if emsa_pss_verify(msg, i2osp(m, emlen), embits, slen) else 2


def raw_sign(sk, em_int):
    """the RSA private operation on an integer: builds signatures over chosen (possibly malformed) encodings"""
    return i2osp(pow(em_int, sk.d, sk.n), sk.klen)


def tampered(k, slen, msg, rng):
    """(label, signature, status) for a valid signature over msg and one signature per EMSA-PSS failure class, built
    with the private key over a tampered encoding, and s = N, s = N + 2"""
    embits = k.n.bit_length() - 1
    emlen = (embits + 7) // 8
    salt = rng.randbytes(slen)
    em = bytearray(emsa_pss_encode(msg, embits, salt))
    dblen = emlen - HLEN - 1
    ps = dblen - slen - 1

    def sig(e):
        return raw_sign(k, os2ip(bytes(e)))

    def flip_db(i, x):
        e = bytearray(em)
        e[i] ^= x
        return sig(e)
    out = [("valid", sig(em), 0)]
    e = bytearray(em)
    e[-1] = 0xbd
    out.append(("trailer", sig(e), 2))
    topbits = 8 * emlen - embits
    if topbits:
        e = bytearray(em)
        e[0] |= 0x80
        out.append(("top bits", sig(e), 2))
    else:  # bitlen(N) = 1 mod 8: the byte above the encoded message must be zero
        out.append(("top byte", raw_sign(k, os2ip(b"\x01" + bytes(em))), 2))
    out.append(("PS", flip_db(ps // 2, 0x10), 2))
    out.append(("0x01", flip_db(ps, 0x03), 2))
    e = bytearray(em)
    e[dblen + 5] ^= 1  # H seeds the MGF1 mask: the unmasked DB is garbage and the PS check fails
    out.append(("H, the MGF1 seed", sig(e), 2))
    # a consistent encoding of another message: every structural check passes and H != H' fails it
    out.append(("H != H'", sig(emsa_pss_encode(msg + b"\x00", embits, salt)), 2))
    if slen:
        out.append(("salt", flip_db(dblen - 1, 0x40), 2))
    out.append(("s = N", i2osp(k.n, k.klen), 1))
    out.append(("s > N", i2osp(k.n + 2, k.klen), 1))
    assert all(verify_status(k, slen, msg, s) == st for _, s, st in out), [
        (n, verify_status(k, slen, msg, s)) for n, s, _ in out]
    return out


# ---------------------------------------------------------------- client
def prepare(variant, msg, prefix):
    return (prefix if VARIANTS[variant][2] else b"") + msg


def blind(pk, variant, prepared, salt, r):
    """(blinded message, inv = r^-1 mod N) of RFC 9474 section 4.2 with the given salt and r"""
    embits = pk.n.bit_length() - 1
    m = os2ip(emsa_pss_encode(prepared, embits, salt))
    assert 0 < m < pk.n
    return i2osp(m * pow(r, pk.e, pk.n) % pk.n, pk.klen), pow(r, -1, pk.n)


def finalize(pk, variant, prepared, blind_sig, inv):
    sig = i2osp(os2ip(blind_sig) * inv % pk.n, pk.klen)
    assert verify_status(pk, VARIANTS[variant][1], prepared, sig) == 0
    return sig


# ---------------------------------------------------------------- fixtures
def rfc_vectors():
    with gzip.open(os.path.join(GOLDEN, "brsa_rfc9474.json.gz")) as f:
        return json.load(f)


def rfc_key():
    v = rfc_vectors()[0]
    return Key(*(int(v[k], 16) for k in ("n", "e", "d", "p", "q")))


def _der_ints(der):
    """the INTEGERs of a PKCS #1 RSAPrivateKey: version, n, e, d, p, q, dp, dq, qinv"""
    def length(i):
        n = der[i]
        if n < 0x80:
            return n, i + 1
        k = n & 0x7f
        return int.from_bytes(der[i + 1:i + 1 + k], "big"), i + 1 + k
    assert der[0] == 0x30
    _, i = length(1)
    out = []
    while i < len(der):
        assert der[i] == 0x02
        n, i = length(i + 1)
        out.append(int.from_bytes(der[i:i + n], "big"))
        i += n
    return out


def pem_key():
    lines = open(os.path.join(GOLDEN, "brsa_rfc9500_2048.pem")).read().split("\n")
    der = base64.b64decode("".join(x for x in lines if x and not x.startswith("-----")))
    _, n, e, d, p, q = _der_ints(der)[:6]
    return Key(n, e, d, p, q)


def derived_keys():
    with gzip.open(os.path.join(GOLDEN, "brsa_keys.json.gz")) as f:
        ks = json.load(f)
    return {name: Key(*(int(v[k], 16) for k in ("n", "e", "d", "p", "q"))) for name, v in ks.items()}


def all_keys():
    """every fixture key by name"""
    return {"rsa2048": pem_key(), **derived_keys(), "rsa4096": rfc_key()}
