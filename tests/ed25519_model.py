"""Ed25519 in Python integers, for the tests: the edwards25519 group law and encoding of RFC 8032 section 5.1, and the
reference's cofactorless verification (sign/ed25519 ed25519.go verify, point.go FromBytes).

Independent of the device code, of the oracle and of OpenSSL.  Verify accepts iff S < L, A decodes (y < p, u / v is a
square, x = 0 only with the sign bit clear) and encode([S] B - [k] A) equals R byte for byte, k = SHA-512(R || A || M)
mod L.  No cofactor is cleared and no encoding is reduced: a torsion component of A is seen through [k] A, one of R
makes the byte comparison fail, and a non-canonical S, A or R is rejected.  `torsion_cases` builds the inputs where
implementations of this rule disagree, each with the verdict the rule gives, checked against the statement that
implies it.

Points are extended coordinates (X, Y, Z, T) with x = X / Z, y = Y / Z, x y = T / Z, so a multiplication costs no
inversion; the affine values are only formed to encode.
"""
from __future__ import annotations

import hashlib
import random

P = 2**255 - 19
L = 2**252 + 27742317777372353535851937790883648493
D = -121665 * pow(121666, P - 2, P) % P
D2 = 2 * D % P
SQRT_M1 = pow(2, (P - 1) // 4, P)
IDENTITY = (0, 1, 1, 0)


def add(p1, p2):
    """The complete addition for a = -1 (add-2008-hwcd-3); also right for p1 = p2 and for the identity."""
    X1, Y1, Z1, T1 = p1
    X2, Y2, Z2, T2 = p2
    a = (Y1 - X1) * (Y2 - X2) % P
    b = (Y1 + X1) * (Y2 + X2) % P
    c = T1 * D2 * T2 % P
    d = 2 * Z1 * Z2 % P
    e, f, g, h = b - a, d - c, d + c, b + a
    return e * f % P, g * h % P, f * g % P, e * h % P


def neg(p1):
    X, Y, Z, T = p1
    return -X % P, Y, Z, -T % P


def mul(k: int, p1):
    r = IDENTITY
    for bit in bin(k)[2:] if k > 0 else "":
        r = add(r, r)
        if bit == "1":
            r = add(r, p1)
    return r


def affine(p1):
    X, Y, Z, _ = p1
    zi = pow(Z, P - 2, P)
    return X * zi % P, Y * zi % P


def encode(p1) -> bytes:
    """point.go ToBytes: canonical y, the low bit of x in bit 255."""
    x, y = affine(p1)
    return (y | (x & 1) << 255).to_bytes(32, "little")


def equal(p1, p2) -> bool:
    return (p1[0] * p2[2] - p2[0] * p1[2]) % P == 0 and (p1[1] * p2[2] - p2[1] * p1[2]) % P == 0


def decode(b: bytes):
    """point.go FromBytes: None for y >= p, for u / v without a square root, and for x = 0 with the sign bit set.
    y is never reduced mod p."""
    if len(b) != 32:
        return None
    v = int.from_bytes(b, "little")
    sign, y = v >> 255, v & (2**255 - 1)
    if y >= P:
        return None
    u, w = (y * y - 1) % P, (D * y * y + 1) % P
    x = u * pow(w, 3, P) * pow(u * pow(w, 7, P), (P - 5) // 8, P) % P
    if (w * x * x - u) % P:
        if (w * x * x + u) % P:
            return None
        x = x * SQRT_M1 % P
    if x == 0 and sign:
        return None
    if x & 1 != sign:
        x = P - x
    return x, y, 1, x * y % P


def on_curve(p1) -> bool:
    x, y = affine(p1)
    return (-x * x + y * y - 1 - D * x * x * y * y) % P == 0


B = decode((4 * pow(5, P - 2, P) % P).to_bytes(32, "little"))  # y = 4/5, x even


def _base_table():
    rows, b = [], B
    for _ in range(64):
        row = [IDENTITY]
        for _ in range(15):
            row.append(add(row[-1], b))
        rows.append(row)
        b = add(row[-1], b)  # [16^(i + 1)] B
    return rows


_BT = _base_table()  # _BT[i][j] = [j 16^i] B


def mul_base(k: int):
    """[k] B for 0 <= k < 2^256, one addition per hexadecimal digit of k."""
    r = IDENTITY
    for i in range(64):
        r = add(r, _BT[i][k >> (4 * i) & 15])
    return r


assert equal(mul_base(L), IDENTITY) and equal(mul_base(2**256 - 1), mul(2**256 - 1, B))


def order(p1) -> int:
    """The order of a point of order dividing 8, else 0."""
    q = p1
    for n in (1, 2, 4, 8):
        if equal(q, IDENTITY):
            return n
        q = add(q, q)
    return 0


def sha512_mod_l(*parts: bytes) -> int:
    return int.from_bytes(hashlib.sha512(b"".join(parts)).digest(), "little") % L


def expand(seed: bytes):
    """(clamped scalar, prefix) of SHA-512(seed) (ed25519.go:431-434)."""
    h = hashlib.sha512(seed).digest()
    a = int.from_bytes(h[:32], "little") & ~7 & (2**255 - 1) | 2**254
    return a, h[32:]


def public(seed: bytes) -> bytes:
    return encode(mul_base(expand(seed)[0]))


def sign(seed: bytes, A: bytes, msg: bytes) -> bytes:
    """Sign (ed25519.go:225-294) with A (32 bytes) as given."""
    a, prefix = expand(seed)
    r = sha512_mod_l(prefix, msg)
    R = encode(mul_base(r))
    k = sha512_mod_l(R, A, msg)
    return R + ((r + k * a) % L).to_bytes(32, "little")


def verify(A: bytes, msg: bytes, sig: bytes) -> bool:
    """verify (ed25519.go:329-368), pure Ed25519."""
    if len(A) != 32 or len(sig) != 64:
        return False
    S = int.from_bytes(sig[32:], "little")
    if S >= L:
        return False
    Ap = decode(A)
    if Ap is None:
        return False
    k = sha512_mod_l(sig[:32], A, msg)
    return encode(add(mul_base(S), mul(k, neg(Ap)))) == sig[:32]


def _torsion():
    """[i] T8 for i = 0..7, T8 = [L] Q of order 8 for the decodable Q = (x, y) with the smallest y >= 2 that gives one."""
    y = 2
    while True:
        Q = decode(y.to_bytes(32, "little"))
        if Q is not None:
            T8 = mul(L, Q)
            if order(T8) == 8:
                break
        y += 1
    pts = [IDENTITY]
    for _ in range(7):
        pts.append(add(pts[-1], T8))
    return pts


TORSION = _torsion()
ORDERS = [8 // (i & -i) if i else 1 for i in range(8)]  # ord([i] T8) = 8 / gcd(i, 8)
assert [order(T) for T in TORSION] == ORDERS
assert all(on_curve(T) for T in TORSION)
assert all(equal(add(TORSION[i], TORSION[j]), TORSION[(i + j) % 8]) for i in range(8) for j in range(8))
assert len({encode(T) for T in TORSION}) == 8
assert affine(TORSION[4]) == (0, P - 1) and {affine(TORSION[2]), affine(TORSION[6])} == {(SQRT_M1, 0), (P - SQRT_M1, 0)}
T2, T4, T8 = TORSION[4], TORSION[2], TORSION[1]  # one point of each order 2, 4, 8


def _le(v: int) -> bytes:
    return v.to_bytes(32, "little")


def _search(base: bytes, k_of, want):
    """The first msg = base || i (two bytes) with want(k_of(msg))."""
    for i in range(1 << 16):
        msg = base + i.to_bytes(2, "little")
        if want(k_of(msg)):
            return msg
    raise AssertionError("no message found")


def torsion_cases(seed: int = 0):
    """(name, pk, msg, sig, verdict) for small-order and mixed-order keys and non-canonical encodings.  Each verdict is
    derived from the statement that implies it (k mod ord(T), y >= p, S >= L, ...) and checked against `verify`."""
    rng = random.Random(seed)
    out = []
    s_edges = [0, 1, L - 1, 2**252, rng.randrange(L)]
    sB = {S: encode(mul_base(S)) for S in s_edges}

    # low-order A = T with R = encode([S] B): Q = [S] B - [k] T, so the signature verifies iff [k] T = O
    for j, T in enumerate(TORSION):
        A, n = encode(T), ORDERS[j]
        for S in s_edges:
            R = sB[S]
            for want in (True, False) if n > 1 else (True,):
                msg = _search(b"low-order %d %d " % (j, want), lambda m: sha512_mod_l(R, A, m), lambda k: (k % n == 0) == want)
                out.append(("low-order A = [%d] T8, S = %#x, %s" % (j, S, want), A, msg, R + _le(S), want))

    # mixed-order A = [a] B + T signed with A as given: R = [r] B, S = r + k a, so Q = R - [k] T
    for n, T in ((2, T2), (4, T4), (8, T8)):
        sd = bytes(rng.randrange(256) for _ in range(32))
        a, prefix = expand(sd)
        A = encode(add(mul_base(a), T))
        for want in (True, False):
            def k_of(m):
                return sha512_mod_l(encode(mul_base(sha512_mod_l(prefix, m))), A, m)
            msg = _search(b"mixed-order %d %d " % (n, want), k_of, lambda k: (k % n == 0) == want)
            out.append(("mixed-order A, ord(T) = %d, %s" % (n, want), A, msg, sign(sd, A, msg), want))

    # R carrying torsion: rejected.  Under a prime-order key k changes with R; under the identity key Q = [S] B does not
    # depend on k, and [8] Q = [8] R still holds, so a cofactored check would accept
    sd = bytes(range(32))
    A = public(sd)
    msg = b"torsion in R"
    sig = sign(sd, A, msg)
    R = decode(sig[:32])
    S0 = int.from_bytes(sig[32:], "little")
    out.append(("valid", A, msg, sig, True))
    ident = encode(IDENTITY)
    for n, T in ((2, T2), (4, T4), (8, T8)):
        out.append(("R + T, ord(T) = %d" % n, A, msg, encode(add(R, T)) + sig[32:], False))
        out.append(("identity A, R = [S] B + T, ord(T) = %d" % n, ident, msg, encode(add(mul_base(S0), T)) + sig[32:], False))

    # non-canonical S: rejected, though S mod L would verify (under the identity key every R = [S mod L] B fits)
    out.append(("S + L", A, msg, sig[:32] + _le(S0 + L), False))
    for S in (L, S0 + L, 2**256 - 1):
        out.append(("identity A, S = %#x" % S, ident, msg, encode(mul_base(S % L)) + _le(S), False))
    out.append(("identity A, S = L - 1", ident, msg, sB[L - 1] + _le(L - 1), True))

    # non-canonical A: every y in [p, 2^255) with either sign bit.  y = p and y = p + 1 reduce to the order-4 points and
    # to the identity; their messages make [k] T = O, so a decoder that reduced y would accept them
    S = s_edges[-1]
    R = sB[S]
    for y in range(P, 2**255):
        for sg in (0, 1):
            A = _le(y | sg << 255)
            T = decode(_le(y - P | sg << 255))
            if T is not None and order(T):
                n = order(T)
                msg = _search(b"y = p + %d " % (y - P), lambda m: sha512_mod_l(R, A, m), lambda k: k % n == 0)
                assert encode(add(mul_base(S), mul(sha512_mod_l(R, A, msg), neg(T)))) == R
            else:
                msg = b"y = p + %d" % (y - P)
            out.append(("A: y = p + %d, sign %d" % (y - P, sg), A, msg, R + _le(S), False))
    # x = 0 with the sign bit: y = 1 (the identity) and y = p - 1 (order 2); the message makes [k] T = O, so dropping
    # the test would accept them
    for name, y, n in (("y = 1", 1, 1), ("y = p - 1", P - 1, 2)):
        A = _le(y | 1 << 255)
        msg = _search(b"x = 0 with sign, " + name.encode(), lambda m: sha512_mod_l(R, A, m), lambda k: k % n == 0)
        out.append(("A: x = 0 with sign, " + name, A, msg, R + _le(S), False))
    y = 2
    while decode(_le(y)) is not None:
        y += 1
    assert decode(_le(y | 1 << 255)) is None
    out.append(("A: y = %d, no square root" % y, _le(y), b"no root", R + _le(S), False))
    # y = 0 with either sign bit: the order-4 points, accepted when [k] T = O
    for sg in (0, 1):
        A = _le(sg << 255)
        assert decode(A) is not None and order(decode(A)) == 4
        msg = _search(b"y = 0, sign %d " % sg, lambda m: sha512_mod_l(R, A, m), lambda k: k % 4 == 0)
        out.append(("A: y = 0, sign %d" % sg, A, msg, R + _le(S), True))

    # non-canonical R: the identity as y = p + 1, and with the sign bit.  Under A = O or A = T8 with [k] T8 = O and S = 0,
    # Q = O, whose canonical encoding would verify
    for name, Rn in (("y = p + 1", _le(P + 1)), ("x = -0", _le(1 | 1 << 255))):
        for A, n in ((ident, 1), (encode(T8), 8)):
            msg = _search(b"R: " + name.encode(), lambda m: sha512_mod_l(Rn, A, m), lambda k: k % n == 0)
            assert encode(add(mul_base(0), mul(sha512_mod_l(Rn, A, msg), neg(decode(A))))) == ident
            out.append(("R: %s, ord(A) = %d" % (name, n), A, msg, Rn + _le(0), False))

    res = []
    for case in out:
        name, pk, msg, sig, want = case[:5]
        assert verify(pk, msg, sig) == want, name
        res.append((name, pk, msg, sig, want))
    return res
