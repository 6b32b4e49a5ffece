"""Ed448 in Python integers, for the tests: the edwards448 group law and encoding of RFC 8032 section 5.2, and the
verification equation of the reference (sign/ed448 verify with goldilocks CombinedMult).

Independent of the device code, of the oracle and of OpenSSL.  The reference computes Q = CombinedMult(S, k, -A) on
the 4-isogenous twist with S / 4 and k / 4 mod l and maps it back, so Q = [S] G - [4 ((k / 4) mod l)] A: the 4-torsion
component of A is dropped.  That is neither RFC 8032's cofactored check nor a plain cofactorless one; `verify` states
it with the plain group law, and the tests compare the device and the oracle against it on torsion inputs.
"""
from __future__ import annotations

import hashlib

P = 2**448 - 2**224 - 1
L = 2**446 - 13818066809895115352007386748515426880336692474882178609894547503885
D = -39081 % P
GX = 224580040295924300187604334099896036246789641632564134246125461686950415467406032909029192869357953282578032075146446173674602635247710
GY = 298819210078481492676017930443930673437544040154080242095928241372331506189835876003536878655418784733982303233503462500531545062832660
G = (GX, GY)
IDENTITY = (0, 1)


def add(p1, p2):
    (x1, y1), (x2, y2) = p1, p2
    t = D * x1 * x2 * y1 * y2 % P
    x3 = (x1 * y2 + y1 * x2) * pow(1 + t, P - 2, P) % P
    y3 = (y1 * y2 - x1 * x2) * pow(1 - t, P - 2, P) % P
    return x3, y3


def neg(p1):
    return (-p1[0] % P, p1[1])


def mul(k, p1):
    r = IDENTITY
    for bit in bin(k)[2:] if k > 0 else "":
        r = add(r, r)
        if bit == "1":
            r = add(r, p1)
    return r


def encode(p1):
    x, y = p1
    return y.to_bytes(56, "little") + bytes([(x & 1) << 7])


def decode(b: bytes):
    """point.go FromBytes: None if byte 56 & 0x7f, y >= p, no square root, or x = 0 with the sign bit set."""
    if len(b) != 57 or b[56] & 0x7F:
        return None
    sign = b[56] >> 7
    y = int.from_bytes(b[:56], "little")
    if y >= P:
        return None
    u, v = (y * y - 1) % P, (D * y * y - 1) % P
    x = u**3 * v * pow(u**5 * v**3, (P - 3) // 4, P) % P
    if (v * x * x - u) % P:
        return None
    if x == 0 and sign:
        return None
    if x & 1 != sign:
        x = P - x
    return x, y


def on_curve(p1):
    x, y = p1
    return (x * x + y * y - 1 - D * x * x * y * y) % P == 0


def dom(ctx: bytes) -> bytes:
    return b"SigEd448" + bytes([0, len(ctx)]) + ctx


def shake(data: bytes) -> int:
    return int.from_bytes(hashlib.shake_256(data).digest(114), "little")


def expand(seed: bytes):
    h = bytearray(hashlib.shake_256(seed).digest(114))
    h[0] &= 0xFC
    h[56] = 0
    h[55] |= 0x80
    return int.from_bytes(h[:57], "little") % L, bytes(h[57:])


def public(seed: bytes) -> bytes:
    return encode(mul(expand(seed)[0], G))


def sign(seed: bytes, A: bytes, msg: bytes, ctx: bytes = b"") -> bytes:
    """signAll with A (57 bytes) as given."""
    s, prefix = expand(seed)
    r = shake(dom(ctx) + prefix + msg) % L
    R = encode(mul(r, G))
    k = shake(dom(ctx) + R + A + msg) % L
    return R + ((r + k * s) % L).to_bytes(57, "little")


def verify(A: bytes, msg: bytes, sig: bytes, ctx: bytes = b"") -> bool:
    if len(sig) != 114 or len(A) != 57 or len(ctx) > 255:
        return False
    S = int.from_bytes(sig[57:], "little")
    if sig[113] != 0 or S >= L:
        return False
    Ap = decode(A)
    if Ap is None:
        return False
    k = shake(dom(ctx) + sig[:57] + A + msg) % L
    k4 = 4 * (k * pow(4, -1, L) % L)
    Q = add(mul(S, G), neg(mul(k4, Ap)))
    return encode(Q) == sig[:57]


# points of order 1, 2 and 4: (0, 1), (0, -1), (1, 0), (-1, 0)
TORSION = [(0, 1), (0, P - 1), (1, 0), (P - 1, 0)]


def torsion_cases(seed_base: int = 0):
    """(name, pk, msg, sig, ctx, verdict) for the torsion and encoding edge cases, with the verdict of `verify` and the
    one the reference's equation implies checked against each other."""
    import random
    rng = random.Random(seed_base)
    out = []
    msg = b"torsion"
    for j, T in enumerate(TORSION):  # low-order public keys accept any R = encode([S] G), for every message
        S = rng.randrange(L)
        sig = encode(mul(S, G)) + S.to_bytes(57, "little")
        out.append(("low-order pk %d" % j, encode(T), msg + bytes([j]), sig, b"", True))
    for j, T in enumerate(TORSION[1:]):  # A_l + T of order 2 and 4, signed with s and the key seed || pk
        seed = bytes(rng.randrange(256) for _ in range(57))
        s = expand(seed)[0]
        pk = encode(add(mul(s, G), T))
        sig = sign(seed, pk, msg)
        out.append(("A + T%d" % (j + 1), pk, msg, sig, b"", True))
        Rt = encode(add(decode(sig[:57]), T))  # R carrying torsion
        out.append(("R + T%d" % (j + 1), pk, msg, Rt + sig[57:], b"", False))
    seed = bytes(range(57))
    pk = public(seed)
    sig = sign(seed, pk, msg)
    S = int.from_bytes(sig[57:], "little")
    out.append(("valid", pk, msg, sig, b"", True))
    out.append(("S + l", pk, msg, sig[:57] + (S + L).to_bytes(57, "little"), b"", False))
    out.append(("S = l", pk, msg, sig[:57] + L.to_bytes(57, "little"), b"", False))
    out.append(("byte 113", pk, msg, sig[:113] + b"\x01", b"", False))
    for name, enc in (("y = p", P.to_bytes(56, "little") + b"\0"), ("y = p + 1", (P + 1).to_bytes(56, "little") + b"\0"),
                      ("byte 56 = 1", pk[:56] + b"\x01"), ("x = 0, sign", (1).to_bytes(56, "little") + b"\x80"),
                      ("x = 0, y = -1, sign", (P - 1).to_bytes(56, "little") + b"\x80")):
        out.append((name, enc, msg, sig, b"", False))
    res = []
    for name, pk_, m, sg, ctx, want in out:
        assert verify(pk_, m, sg, ctx) == want, name
        res.append((name, pk_, m, sg, ctx, want))
    return res
