"""CPU: the Ed25519 / Ed25519-Dilithium2 oracle (oracle/ed25519.c) against the reference's RFC 8032, sign.input and
Wycheproof vectors, OpenSSL's Ed25519 and hashlib, the composite rebuilt from OpenSSL Ed25519 + hashlib SHAKE256 +
the oracle's round-3 Dilithium2, and the Python-integer model (tests/ed25519_model.py) on small-order and mixed-order
keys and non-canonical encodings."""
import hashlib
import random

import pytest

import ed25519_model as M
from conftest import load_golden

L = 2**252 + 27742317777372353535851937790883648493


@pytest.fixture(scope="module")
def oe():
    from oracle import ed25519
    ed25519.build()
    return ed25519


def _ossl(seed):
    from cryptography.hazmat.primitives.asymmetric.ed25519 import Ed25519PrivateKey
    return Ed25519PrivateKey.from_private_bytes(seed)


def test_sha512_against_hashlib(oe):
    rng = random.Random(1)
    for n in [0, 1, 111, 112, 113, 127, 128, 129, 239, 240, 255, 256, 1000]:
        m = bytes(rng.randrange(256) for _ in range(n))
        assert oe.sha512(m) == hashlib.sha512(m).digest()


def test_reference_vectors(oe):
    v = load_golden("ed25519_vectors.json.gz")
    assert len(v["rfc8032"]) == 5 and len(v["sign_input"]) == 1024 and len(v["wycheproof"]) == 145
    for t in v["rfc8032"] + v["sign_input"]:
        seed, msg = bytes.fromhex(t["seed"]), bytes.fromhex(t["msg"])
        pk, sk = oe.ed25519_keygen(seed)
        assert pk.hex() == t["pk"]
        sig = oe.ed25519_sign(sk, msg)
        assert sig.hex() == t["sig"] and oe.ed25519_verify(pk, msg, sig)
    for t in v["wycheproof"]:
        pk, sk = oe.ed25519_keygen(bytes.fromhex(t["seed"]))
        assert pk.hex() == t["pk"]
        msg, sig = bytes.fromhex(t["msg"]), bytes.fromhex(t["sig"])
        if t["valid"]:
            assert oe.ed25519_sign(sk, msg) == sig
        assert oe.ed25519_verify(pk, msg, sig) == t["valid"], t["tcId"]


def test_against_openssl(oe):
    rng = random.Random(2)
    for i, n in enumerate([0, 1, 111, 112, 127, 128, 239, 240, 10000] * 4):
        seed = bytes(rng.randrange(256) for _ in range(32))
        msg = bytes(rng.randrange(256) for _ in range(n))
        k = _ossl(seed)
        pk, sk = oe.ed25519_keygen(seed)
        assert pk == k.public_key().public_bytes_raw()
        sig = oe.ed25519_sign(sk, msg)
        assert sig == k.sign(msg) and oe.ed25519_verify(pk, msg, sig)
        bad = bytearray(sig)
        bad[rng.randrange(64)] ^= 1 << rng.randrange(8)
        assert not oe.ed25519_verify(pk, msg, bytes(bad))
        s_plus_l = sig[:32] + (int.from_bytes(sig[32:], "little") + L).to_bytes(32, "little")
        assert not oe.ed25519_verify(pk, msg, s_plus_l)


def test_public_half_of_the_key_is_used_as_given(oe):
    seed, other = bytes(range(32)), bytes(range(1, 33))
    wrong = _ossl(other).public_key().public_bytes_raw()
    sig = oe.ed25519_sign(seed + wrong, b"m")
    h = hashlib.sha512(seed).digest()
    a = int.from_bytes(h[:32], "little") & ~7 & (2**255 - 1) | 2**254
    r = int.from_bytes(hashlib.sha512(h[32:] + b"m").digest(), "little") % L
    R = _ossl(seed).sign(b"m")[:32]
    k = int.from_bytes(hashlib.sha512(R + wrong + b"m").digest(), "little") % L
    assert sig == R + ((r + k * a) % L).to_bytes(32, "little")


def test_eddilithium2_rebuilt_from_parts(oe):
    import oracle
    rng = random.Random(3)
    for n in (0, 1, 33, 200):
        seed = bytes(rng.randrange(256) for _ in range(32))
        msg = bytes(rng.randrange(256) for _ in range(n))
        ex = hashlib.shake_256(seed).digest(64)
        dpk, dsk = oracle.mldsa_keygen(2, ex[:32])
        epk = _ossl(ex[32:]).public_key().public_bytes_raw()
        pk, sk = oe.eddilithium2_keygen(seed)
        assert (pk, sk) == (dpk + epk, dsk + ex[32:])
        sig = oe.eddilithium2_sign(sk, msg)
        assert sig == oracle.mldsa_sign(2, dsk, msg)[0] + _ossl(ex[32:]).sign(msg)
        assert oe.eddilithium2_verify(pk, msg, sig)
        for pos in (10, 2430, 2483):
            bad = bytearray(sig)
            bad[pos] ^= 1
            assert not oe.eddilithium2_verify(pk, msg, bytes(bad))
        assert not oe.eddilithium2_verify(pk, msg, sig[:-1])


@pytest.fixture(scope="module")
def cases():
    return M.torsion_cases()


def test_model_against_openssl_and_vectors():
    """The model's public / sign equal OpenSSL's on random seeds, its verify accepts them and rejects a flipped bit,
    and it gives every Wycheproof verdict."""
    rng = random.Random(8)
    for n in (0, 1, 64, 200):
        seed = bytes(rng.randrange(256) for _ in range(32))
        msg = bytes(rng.randrange(256) for _ in range(n))
        k = _ossl(seed)
        A = M.public(seed)
        assert A == k.public_key().public_bytes_raw()
        sig = M.sign(seed, A, msg)
        assert sig == k.sign(msg) and M.verify(A, msg, sig)
        assert not M.verify(A, msg, sig[:7] + bytes([sig[7] ^ 4]) + sig[8:])
    for t in load_golden("ed25519_vectors.json.gz")["wycheproof"]:
        assert M.verify(bytes.fromhex(t["pk"]), bytes.fromhex(t["msg"]), bytes.fromhex(t["sig"])) == t["valid"], t["tcId"]


def test_torsion_cases_cover_every_order(cases):
    """Low-order keys of every order, mixed-order keys with T of order 2, 4 and 8, both verdicts for each nonzero
    order, and all 38 encodings with y >= p."""
    low, mixed = {}, {}
    for name, pk, msg, sig, want in cases:
        A = M.decode(pk)
        if A is None:
            continue
        n = M.order(A)
        if n:
            low.setdefault(n, set()).add(want)
        elif M.order(M.mul(M.L, A)) > 1:
            mixed.setdefault(M.order(M.mul(M.L, A)), set()).add(want)
    assert set(low) == {1, 2, 4, 8} and all(low[n] == {True, False} for n in (2, 4, 8))
    assert mixed == {2: {True, False}, 4: {True, False}, 8: {True, False}}
    big = {pk for _, pk, _, _, _ in cases if int.from_bytes(pk, "little") & (2**255 - 1) >= M.P}
    assert len(big) == 38


def test_torsion_cases(oe, cases):
    """The oracle gives the model's verdict on every small-order, mixed-order and non-canonical case."""
    got = [oe.ed25519_verify(pk, msg, sig) for _, pk, msg, sig, _ in cases]
    assert got == [c[4] for c in cases], [c[0] for c, g in zip(cases, got) if g != c[4]]


def test_eddilithium2_torsion_cases(oe, cases):
    """With a valid Dilithium2 half, the composite's verdict is the model's verdict on the Ed25519 half; with a
    corrupted one it is false."""
    import oracle
    dpk, dsk = oracle.mldsa_keygen(2, bytes(range(32)))
    got = []
    for name, pk, msg, sig, want in cases:
        dsig = oracle.mldsa_sign(2, dsk, msg)[0]
        got.append(oe.eddilithium2_verify(dpk + pk, msg, dsig + sig))
        if want:
            bad = bytearray(dsig)
            bad[100] ^= 1
            assert not oe.eddilithium2_verify(dpk + pk, msg, bytes(bad) + sig), name
    assert got == [c[4] for c in cases]
