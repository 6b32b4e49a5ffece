"""A Python model of RFC 9497's OPRF over the NIST curves (suites P256-SHA256, P384-SHA384, P521-SHA512), server and
client, for the tests: the reference's oprf/{oprf,server,client,keys}.go, zk/dleq/dleq.go, group/short.go and
expander/expander.go restated on Python integers and hashlib.  The reference computes with math/big; this model uses
Jacobian coordinates (a = -3) so that P-521 stays fast, and shares no arithmetic with the device code.

Also: expand_message_xmd, hash_to_field and hash_to_curve (RFC 9380, the SSWU_RO_ suites), with intermediates.
"""
import hashlib
from dataclasses import dataclass

from nistp_model import P384 as _C384, P521 as _C521

BASE, VERIFIABLE, PARTIAL = 0, 1, 2


@dataclass(frozen=True)
class Suite:
    identifier: str
    bits: int
    p: int
    n: int
    b: int
    g: tuple
    hash: object  # hashlib constructor
    L: int        # hash_to_field bytes per element
    Z: int        # the SSWU Z (negative)

    @property
    def nbytes(self):
        return (self.bits + 7) // 8

    Ns = nbytes

    @property
    def Ne(self):
        return 1 + self.nbytes

    @property
    def Nh(self):
        return self.hash().digest_size

    @property
    def proof_size(self):
        return 2 * self.nbytes


P256 = Suite(
    "P256-SHA256", 256, 2**256 - 2**224 + 2**192 + 2**96 - 1,
    0xffffffff00000000ffffffffffffffffbce6faada7179e84f3b9cac2fc632551,
    0x5ac635d8aa3a93e7b3ebbd55769886bc651d06b0cc53b0f63bce3c3e27d2604b,
    (0x6b17d1f2e12c4247f8bce6e563a440f277037d812deb33a0f4a13945d898c296,
     0x4fe342e2fe1a7f9b8ee7eb4a7c0f9e162bce33576b315ececbb6406837bf51f5),
    hashlib.sha256, 48, -10)
P384 = Suite("P384-SHA384", 384, _C384.p, _C384.n, _C384.b, _C384.g, hashlib.sha384, 72, -12)
P521 = Suite("P521-SHA512", 521, _C521.p, _C521.n, _C521.b, _C521.g, hashlib.sha512, 98, -4)
SUITES = {s.identifier: s for s in (P256, P384, P521)}


def i2osp(v: int, n: int) -> bytes:
    return v.to_bytes(n, "big")


# ---------------------------------------------------------------- group: Jacobian (X, Y, Z), x = X / Z^2, y = Y / Z^3
def _jdbl(s, P1):
    X, Y, Z = P1
    if Z == 0 or Y == 0:
        return (1, 1, 0)
    p = s.p
    d, g = Z * Z % p, Y * Y % p
    beta = X * g % p
    alpha = 3 * (X - d) * (X + d) % p
    X3 = (alpha * alpha - 8 * beta) % p
    Z3 = ((Y + Z) ** 2 - g - d) % p
    Y3 = (alpha * (4 * beta - X3) - 8 * g * g) % p
    return (X3, Y3, Z3)


def _jadd(s, P1, P2):
    if P1[2] == 0:
        return P2
    if P2[2] == 0:
        return P1
    p = s.p
    X1, Y1, Z1 = P1
    X2, Y2, Z2 = P2
    z1, z2 = Z1 * Z1 % p, Z2 * Z2 % p
    U1, U2 = X1 * z2 % p, X2 * z1 % p
    S1, S2 = Y1 * Z2 * z2 % p, Y2 * Z1 * z1 % p
    if U1 == U2:
        return _jdbl(s, P1) if S1 == S2 else (1, 1, 0)
    H, R = (U2 - U1) % p, (S2 - S1) % p
    H2 = H * H % p
    H3 = H * H2 % p
    V = U1 * H2 % p
    X3 = (R * R - H3 - 2 * V) % p
    return (X3, (R * (V - X3) - S1 * H3) % p, Z1 * Z2 * H % p)


def _affine(s, P1):
    if P1[2] == 0:
        return None
    zi = pow(P1[2], -1, s.p)
    z2 = zi * zi % s.p
    return (P1[0] * z2 % s.p, P1[1] * z2 * zi % s.p)


def _jac(pt):
    return (1, 1, 0) if pt is None else (pt[0], pt[1], 1)


def add(s, a, b):
    """a + b on affine points (None = the identity)."""
    return _affine(s, _jadd(s, _jac(a), _jac(b)))


def mul(s, k, pt):
    """[k] pt, with a 4-bit fixed window."""
    k %= s.n
    if pt is None or k == 0:
        return None
    tab = [(1, 1, 0), _jac(pt)]
    for _ in range(14):
        tab.append(_jadd(s, tab[-1], tab[1]))
    r = (1, 1, 0)
    for i in range((k.bit_length() + 3) // 4 - 1, -1, -1):
        for _ in range(4):
            r = _jdbl(s, r)
        r = _jadd(s, r, tab[(k >> (4 * i)) & 15])
    return _affine(s, r)


def on_curve(s, pt) -> bool:
    x, y = pt
    return (y * y - (x * x * x - 3 * x + s.b)) % s.p == 0


def compress(s, pt) -> bytes:
    """MarshalBinaryCompress: 0x02 | 0x03 || X (the identity, which the server never outputs, is 0x00)."""
    if pt is None:
        return b"\x00"
    return bytes([2 | (pt[1] & 1)]) + i2osp(pt[0], s.nbytes)


def decompress(s, b: bytes):
    """UnmarshalBinary on a compressed row of Ne bytes: the point, or None for a bad prefix, X >= p or no square root."""
    if len(b) != s.Ne or b[0] not in (2, 3):
        return None
    x = int.from_bytes(b[1:], "big")
    if x >= s.p:
        return None
    rhs = (x * x * x - 3 * x + s.b) % s.p
    y = pow(rhs, (s.p + 1) // 4, s.p)
    if y * y % s.p != rhs:
        return None
    if (y & 1) != (b[0] & 1):
        y = (s.p - y) % s.p
    return (x, y)


# ---------------------------------------------------------------- RFC 9380
def expand_message_xmd(hashf, msg: bytes, dst: bytes, n: int) -> bytes:
    h = hashf()
    bl, sl = h.digest_size, h.block_size
    if len(dst) > 255:
        dst = hashf(b"H2C-OVERSIZE-DST-" + dst).digest()
    ell = (n + bl - 1) // bl
    assert ell <= 255 and n < 65536
    dst_prime = dst + bytes([len(dst)])
    b0 = hashf(bytes(sl) + msg + i2osp(n, 2) + b"\x00" + dst_prime).digest()
    bi = hashf(b0 + b"\x01" + dst_prime).digest()
    out = bi
    for i in range(2, ell + 1):
        bi = hashf(bytes(a ^ c for a, c in zip(b0, bi)) + bytes([i]) + dst_prime).digest()
        out += bi
    return out[:n]


def hash_to_field(s, msg: bytes, dst: bytes, count: int, modulus: int):
    u = expand_message_xmd(s.hash, msg, dst, count * s.L)
    return [int.from_bytes(u[i * s.L:(i + 1) * s.L], "big") % modulus for i in range(count)]


def _is_square(s, v):
    return pow(v, (s.p - 1) // 2, s.p) in (0, 1)


def sswu(s, u: int):
    """map_to_curve_simple_swu (RFC 9380 section 6.6.2) for A = -3."""
    p, A, B, Z = s.p, s.p - 3, s.b, s.Z % s.p
    tv1 = (Z * Z * pow(u, 4, p) + Z * u * u) % p
    if tv1 == 0:
        x1 = B * pow(Z * A, -1, p) % p
    else:
        x1 = (-B * pow(A, -1, p)) * (1 + pow(tv1, -1, p)) % p
    gx1 = (x1 ** 3 + A * x1 + B) % p
    x2 = Z * u * u * x1 % p
    gx2 = (x2 ** 3 + A * x2 + B) % p
    x, y = (x1, pow(gx1, (p + 1) // 4, p)) if _is_square(s, gx1) else (x2, pow(gx2, (p + 1) // 4, p))
    if (u & 1) != (y & 1):
        y = (p - y) % p
    return (x, y)


def hash_to_curve(s, msg: bytes, dst: bytes):
    """(u0, u1), Q0, Q1, P of the SSWU_RO_ suite (the cofactor is 1)."""
    u = hash_to_field(s, msg, dst, 2, s.p)
    q0, q1 = sswu(s, u[0]), sswu(s, u[1])
    return u, q0, q1, add(s, q0, q1)


# ---------------------------------------------------------------- RFC 9497
def context(s, mode: int) -> bytes:
    return b"OPRFV1-" + bytes([mode]) + b"-" + s.identifier.encode()


def hash_to_group(s, mode, msg):
    return hash_to_curve(s, msg, b"HashToGroup-" + context(s, mode))[3]


def hash_to_scalar(s, mode, msg, dst=None):
    return hash_to_field(s, msg, dst or b"HashToScalar-" + context(s, mode), 1, s.n)[0]


def derive_key(s, mode, seed: bytes, info: bytes):
    """keys.go:103-132: (sk as Ns bytes, pk as Ne bytes)."""
    assert len(seed) == 32 and len(info) < 65536
    din = seed + i2osp(len(info), 2) + info
    for ctr in range(256):
        sk = hash_to_scalar(s, mode, din + bytes([ctr]), b"DeriveKeyPair" + context(s, mode))
        if sk:
            return i2osp(sk, s.Ns), compress(s, mul(s, sk, s.g))
    raise AssertionError("DeriveKeyPair")


def info_scalar(s, info: bytes) -> int:
    """scalarFromInfo (mode 2)."""
    return hash_to_scalar(s, PARTIAL, b"Info" + i2osp(len(info), 2) + info)


def _weights(s, mode, Y, bencs, cencs):
    """The composite weights d_j of ComputeComposites for the compressed B_j and C_j."""
    bm = compress(s, Y)
    sdst = b"Seed-" + context(s, mode)
    seed = s.hash(i2osp(len(bm), 2) + bm + i2osp(len(sdst), 2) + sdst).digest()
    return [hash_to_scalar(s, mode, i2osp(len(seed), 2) + seed + i2osp(j, 2) + i2osp(len(bj), 2) + bj
                           + i2osp(len(cj), 2) + cj + b"Composite") for j, (bj, cj) in enumerate(zip(bencs, cencs))]


def _composites(s, mode, k, Y, Bs, Cs):
    """(M, Z) of ComputeComposites; with k, Z = [k] M (the prover's shortcut), else Z = sum d_j C_j."""
    ds = _weights(s, mode, Y, [compress(s, b) for b in Bs], [compress(s, c) for c in Cs])
    M = Z = None
    for d, b, c in zip(ds, Bs, Cs):
        M = add(s, M, mul(s, d, b))
        if k is None:
            Z = add(s, Z, mul(s, d, c))
    if k is not None:
        Z = mul(s, k, M)
    return M, Z


def _challenge(s, mode, pts):
    data = b""
    for pt in pts:
        e = compress(s, pt)
        data += i2osp(len(e), 2) + e
    return hash_to_scalar(s, mode, data + b"Challenge")


def prove(s, mode, k, Y, Bs, Cs, r):
    """ProveBatchWithRandomnessRFC9497(k, Y = [k]G, B, C = [k]B, r): c || s."""
    M, Z = _composites(s, mode, k, Y, Bs, Cs)
    c = _challenge(s, mode, [Y, M, Z, mul(s, r, s.g), mul(s, r, M)])
    return i2osp(c, s.Ns) + i2osp((r - c * k) % s.n, s.Ns)


def verify(s, mode, Y, Bs, Cs, proof: bytes) -> bool:
    c, sc = int.from_bytes(proof[:s.Ns], "big"), int.from_bytes(proof[s.Ns:], "big")
    if c >= s.n or sc >= s.n:
        return False
    M, Z = _composites(s, mode, None, Y, Bs, Cs)
    t2 = add(s, mul(s, sc, s.g), mul(s, c, Y))
    t3 = add(s, mul(s, sc, M), mul(s, c, Z))
    return _challenge(s, mode, [Y, M, Z, t2, t3]) == c


class OprfError(Exception):
    def __init__(self, status):
        super().__init__(f"status {status}")
        self.status = status


def _secret(s, mode, k, info):
    """(the proof's key, the evaluation key): (k, k) or (t, t^-1) for mode 2."""
    if mode != PARTIAL:
        return k, k
    t = (k + info_scalar(s, info)) % s.n
    if t == 0:
        raise OprfError(8)
    return t, pow(t, -1, s.n)


def evaluate(s, mode, sk: bytes, blinded, r: bytes = None, info: bytes = b""):
    """server.go:23-85 on one request: (list of evaluated elements, proof bytes or None).  Raises OprfError with the
    device status bits."""
    k = int.from_bytes(sk, "big")
    Bs = [decompress(s, b) for b in blinded]
    st = (1 if any(b is None for b in Bs) else 0) | (0 if 0 < k < s.n else 2)
    rv = int.from_bytes(r, "big") if r is not None else 1
    if mode != BASE and not 0 < rv < s.n:
        st |= 4
    if st:
        raise OprfError(st)
    kp, ke = _secret(s, mode, k, info)
    Ds = [mul(s, ke, b) for b in Bs]
    ev = [compress(s, d) for d in Ds]
    if mode == BASE:
        return ev, None
    if mode == VERIFIABLE:
        return ev, prove(s, mode, kp, mul(s, kp, s.g), Bs, Ds, rv)
    return ev, prove(s, mode, kp, mul(s, kp, s.g), Ds, Bs, rv)


def evaluate_grouped(s, mode, sk: bytes, blinded, r: bytes = None, info: bytes = b""):
    """evaluate() for requests whose m elements come from a few distinct ones: one [ke] B per distinct B, and
    M = sum over distinct b of (sum of the d_j with B_j = b mod n) b, so the weights are still hashed per element but
    there are only as many scalar multiplications as distinct elements.  The same results and errors as evaluate()."""
    k = int.from_bytes(sk, "big")
    pts = {b: decompress(s, b) for b in dict.fromkeys(bytes(b) for b in blinded)}
    st = (1 if any(p is None for p in pts.values()) else 0) | (0 if 0 < k < s.n else 2)
    rv = int.from_bytes(r, "big") if r is not None else 1
    if mode != BASE and not 0 < rv < s.n:
        st |= 4
    if st:
        raise OprfError(st)
    kp, ke = _secret(s, mode, k, info)
    D = {b: mul(s, ke, p) for b, p in pts.items()}
    enc = {b: compress(s, d) for b, d in D.items()}
    ev = [enc[bytes(b)] for b in blinded]
    if mode == BASE:
        return ev, None
    Y = mul(s, kp, s.g)
    # mode 1 proves D = [k]B; mode 2 proves B = [t]D, with the roles of B and D swapped
    benc = [bytes(b) for b in blinded]
    ds = _weights(s, mode, Y, benc, ev) if mode == VERIFIABLE else _weights(s, mode, Y, ev, benc)
    w = dict.fromkeys(pts, 0)
    for b, d in zip(benc, ds):
        w[b] = (w[b] + d) % s.n
    M = None
    for b, wb in w.items():
        M = add(s, M, mul(s, wb, pts[b] if mode == VERIFIABLE else D[b]))
    c = _challenge(s, mode, [Y, M, mul(s, kp, M), mul(s, rv, s.g), mul(s, rv, M)])
    return ev, i2osp(c, s.Ns) + i2osp((rv - c * kp) % s.n, s.Ns)


def finalize_hash(s, mode, inp: bytes, info: bytes, elem: bytes) -> bytes:
    data = i2osp(len(inp), 2) + inp
    if mode == PARTIAL:
        data += i2osp(len(info), 2) + info
    return s.hash(data + i2osp(len(elem), 2) + elem + b"Finalize").digest()


def full_evaluate(s, mode, sk: bytes, inp: bytes, info: bytes = b"") -> bytes:
    """server.go:97-117."""
    k = int.from_bytes(sk, "big")
    if not 0 < k < s.n:
        raise OprfError(2)
    _, ke = _secret(s, mode, k, info)
    E = mul(s, ke, hash_to_group(s, mode, inp))
    return finalize_hash(s, mode, inp, info, compress(s, E))


# ---------------------------------------------------------------- the client (client.go)
def blind(s, mode, inp: bytes, bl: int) -> bytes:
    return compress(s, mul(s, bl, hash_to_group(s, mode, inp)))


def client_verify(s, mode, pk: bytes, blinded, evaluated, proof: bytes, info: bytes = b"") -> bool:
    Bs = [decompress(s, b) for b in blinded]
    Ds = [decompress(s, d) for d in evaluated]
    Y = decompress(s, pk)
    if mode == VERIFIABLE:
        return verify(s, mode, Y, Bs, Ds, proof)
    T = add(s, Y, mul(s, info_scalar(s, info), s.g))
    return verify(s, mode, T, Ds, Bs, proof)


def finalize(s, mode, inp: bytes, bl: int, evaluated: bytes, info: bytes = b"") -> bytes:
    N = mul(s, pow(bl, -1, s.n), decompress(s, evaluated))
    return finalize_hash(s, mode, inp, info, compress(s, N))
