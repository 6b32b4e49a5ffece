"""An independent model of FrodoKEM-640-SHAKE (as the reference's kem/frodo/frodo640shake computes it), built from numpy
and hashlib.shake_128.  OpenSSL has no FrodoKEM, so this model is the second implementation the oracle and the GPU are
checked against.  Matrices are int64 arrays reduced mod 2^16 after each product.
"""
from __future__ import annotations

import hashlib

import numpy as np

N, NBAR, LOGQ = 640, 8, 15
QMASK = (1 << LOGQ) - 1
PK, SK, CT, SS = 9616, 19888, 9720, 16
CDF = np.array([4643, 13363, 20579, 25843, 29227, 31145, 32103, 32525, 32689, 32745, 32762, 32766], dtype=np.int64)


def shake(n: int, *parts: bytes) -> bytes:
    return hashlib.shake_128(b"".join(parts)).digest(n)


def u16(b: bytes) -> np.ndarray:
    return np.frombuffer(b, dtype="<u2").astype(np.int64)


def sample(r: np.ndarray) -> np.ndarray:
    """The CDF sampler: the count of table entries below r >> 1, negated when bit 0 is set (mod 2^16)."""
    r = np.asarray(r, dtype=np.int64)
    g = (CDF[None, :] < (r[..., None] >> 1)).sum(axis=-1) if r.ndim else int((CDF < (r >> 1)).sum())
    return np.where(r & 1, -g, g) & 0xFFFF


def pack(v) -> bytes:
    """15-bit big-endian bit string of the coefficients (mod 2^15)."""
    v = np.asarray(v, dtype=np.int64).reshape(-1) & QMASK
    bits = ((v[:, None] >> np.arange(14, -1, -1)) & 1).astype(np.uint8).reshape(-1)
    return np.packbits(bits).tobytes()


def unpack(b: bytes) -> np.ndarray:
    bits = np.unpackbits(np.frombuffer(b, dtype=np.uint8)).reshape(-1, 15).astype(np.int64)
    return (bits << np.arange(14, -1, -1)).sum(axis=1)


def encode(mu: bytes) -> np.ndarray:
    bits = np.unpackbits(np.frombuffer(mu, dtype=np.uint8), bitorder="little").reshape(64, 2).astype(np.int64)
    return (bits[:, 0] + 2 * bits[:, 1]) << (LOGQ - 2)


def decode(w) -> bytes:
    q = (((np.asarray(w, dtype=np.int64).reshape(-1) & QMASK) + (1 << (LOGQ - 3))) >> (LOGQ - 2)) & 3
    bits = np.stack([q & 1, q >> 1], axis=1).reshape(-1).astype(np.uint8)
    return np.packbits(bits, bitorder="little").tobytes()


def expand_a(seed_a: bytes) -> np.ndarray:
    return np.stack([u16(shake(2 * N, i.to_bytes(2, "little"), seed_a)) for i in range(N)])


def keygen(seed: bytes):
    s, seed_se, z = seed[:16], seed[16:32], seed[32:48]
    seed_a = shake(16, z)
    r = sample(u16(shake(4 * N * NBAR, b"\x5f", seed_se)))
    st, e = r[:N * NBAR].reshape(NBAR, N), r[N * NBAR:].reshape(N, NBAR)
    b = (expand_a(seed_a) @ st.T + e) & 0xFFFF
    pk = seed_a + pack(b)
    sk = s + pk + st.astype("<u2").tobytes() + shake(16, pk)
    return pk, sk


def _reencrypt(seed_a: bytes, b: np.ndarray, hpk: bytes, mu: bytes):
    g2 = shake(32, hpk, mu)
    r = sample(u16(shake(2 * (2 * N * NBAR + 64), b"\x96", g2[:16])))
    sp, ep, epp = r[:N * NBAR].reshape(NBAR, N), r[N * NBAR:2 * N * NBAR].reshape(NBAR, N), r[2 * N * NBAR:].reshape(8, 8)
    bp = (sp @ expand_a(seed_a) + ep) & 0xFFFF
    c = ((sp @ b + epp) + encode(mu).reshape(8, 8)) & QMASK
    return bp, c, g2[16:]


def encaps(pk: bytes, mu: bytes):
    b = unpack(pk[16:]).reshape(N, NBAR)
    bp, c, k = _reencrypt(pk[:16], b, shake(16, pk), mu)
    ct = pack(bp) + pack(c)
    return ct, shake(16, ct, k)


def decaps(sk: bytes, ct: bytes) -> bytes:
    s, pk, st, hpk = sk[:16], sk[16:16 + PK], u16(sk[16 + PK:16 + PK + 2 * N * NBAR]).reshape(NBAR, N), sk[-16:]
    bp, c = unpack(ct[:9600]).reshape(NBAR, N), unpack(ct[9600:]).reshape(8, 8)
    mu = decode((c - bp @ st.T) & QMASK)
    bbp, cc, k = _reencrypt(pk[:16], unpack(pk[16:]).reshape(N, NBAR), hpk, mu)
    ok = np.array_equal(bbp & QMASK, bp) and np.array_equal(cc, c)
    return shake(16, ct, k if ok else s)


def kat_hash(keygen_fn, encaps_fn, decaps_fn, rounds: int = 100, name: str = "FrodoKEM-640-SHAKE") -> str:
    """SHA-256 of the PQCgenKAT transcript of kem/frodo/kat_test.go (seeds from the NIST DRBG).  The three functions
    take and return lists of byte strings: keygen(kseeds) -> (pks, sks), encaps(pks, eseeds) -> (cts, sss),
    decaps(sks, cts) -> sss, so a batched implementation computes all rounds in one call each."""
    from nist_drbg import DRBG
    g = DRBG(bytes(range(48)))
    seeds, kseeds, eseeds = [], [], []
    for _ in range(rounds):
        seed = g.fill(48)
        g2 = DRBG(seed)
        seeds.append(seed)
        kseeds.append(g2.fill(48))
        eseeds.append(g2.fill(16))
    pks, sks = keygen_fn(kseeds)
    cts, sss = encaps_fn(pks, eseeds)
    assert decaps_fn(sks, cts) == sss
    f = hashlib.sha256()
    f.update(f"# {name}\n\n".encode())
    for i in range(rounds):
        f.update(f"count = {i}\nseed = {seeds[i].hex().upper()}\n".encode())
        f.update(f"pk = {pks[i].hex().upper()}\nsk = {sks[i].hex().upper()}\n".encode())
        f.update(f"ct = {cts[i].hex().upper()}\nss = {sss[i].hex().upper()}\n\n".encode())
    return f.hexdigest()
