"""CPU: the Ed25519 / Ed25519-Dilithium2 oracle (oracle/ed25519.c) against the reference's RFC 8032, sign.input and
Wycheproof vectors, OpenSSL's Ed25519 and hashlib, and the composite rebuilt from OpenSSL Ed25519 + hashlib SHAKE256 +
the oracle's round-3 Dilithium2."""
import hashlib
import random

import pytest

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
