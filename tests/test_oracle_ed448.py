"""CPU-only: the Ed448 / Ed448-Dilithium3 oracle (oracle/ed448.c) against the reference's RFC 8032 and Wycheproof
vectors, OpenSSL's Ed448 (empty context) on random seeds and message lengths across the 136-byte SHAKE256 rate, the
Python model of the reference's verification equation on torsion and encoding edge cases, and Ed448-Dilithium3
rebuilt from OpenSSL Ed448, hashlib's SHAKE256 and the oracle's round-3 Dilithium3."""
import hashlib
import random

import pytest

import ed448_model as M
from conftest import load_golden


@pytest.fixture(scope="module")
def oe():
    from oracle import ed448
    return ed448


def test_rfc8032_vectors(oe):
    v = load_golden("ed448_vectors.json.gz")
    assert len(v["rfc8032"]) == 9 and sum(1 for t in v["rfc8032"] if t["ctx"]) == 1
    for t in v["rfc8032"]:
        seed, pk, msg, sig, ctx = (bytes.fromhex(t[k]) for k in ("seed", "pk", "msg", "sig", "ctx"))
        assert oe.ed448_keygen(seed) == (pk, seed + pk)
        assert oe.ed448_sign(seed + pk, msg, ctx) == sig
        assert oe.ed448_verify(pk, msg, sig, ctx)
        assert not oe.ed448_verify(pk, msg, sig, ctx + b"x")


def test_wycheproof_vectors(oe):
    w = load_golden("ed448_vectors.json.gz")["wycheproof"]
    assert len(w) == 86
    for t in w:
        pk, msg, sig = (bytes.fromhex(t[k]) for k in ("pk", "msg", "sig"))
        assert oe.ed448_verify(pk, msg, sig) == t["valid"], t["tcId"]
        if t["valid"]:
            seed = bytes.fromhex(t["seed"])
            assert oe.ed448_keygen(seed)[0] == pk and oe.ed448_sign(seed + pk, msg) == sig


def test_against_openssl(oe):
    from cryptography.hazmat.primitives.asymmetric.ed448 import Ed448PrivateKey
    rng = random.Random(1)
    for n in [0, 1, 2, 24, 25, 26, 60, 66, 67, 68, 69, 70, 78, 79, 80, 135, 136, 137, 271, 272, 273, 1000]:
        seed = bytes(rng.randrange(256) for _ in range(57))
        msg = bytes(rng.randrange(256) for _ in range(n))
        k = Ed448PrivateKey.from_private_bytes(seed)
        pk, sk = oe.ed448_keygen(seed)
        assert pk == k.public_key().public_bytes_raw()
        sig = oe.ed448_sign(sk, msg)
        assert sig == k.sign(msg)
        assert oe.ed448_verify(pk, msg, sig)


def test_context_rules(oe):
    seed = bytes(range(57))
    pk, sk = oe.ed448_keygen(seed)
    for ctx in (b"", b"\0", bytes(range(255))):
        sig = oe.ed448_sign(sk, b"m", ctx)
        assert sig == M.sign(seed, pk, b"m", ctx)
        assert oe.ed448_verify(pk, b"m", sig, ctx) and M.verify(pk, b"m", sig, ctx)
    with pytest.raises(ValueError):
        oe.ed448_sign(sk, b"m", bytes(256))
    assert not oe.ed448_verify(pk, b"m", oe.ed448_sign(sk, b"m"), bytes(256))


def test_torsion_and_encoding_edge_cases(oe):
    """Verdicts of the reference's equation, computed with Python integers (tests/ed448_model.py)."""
    for name, pk, msg, sig, ctx, want in M.torsion_cases():
        assert oe.ed448_verify(pk, msg, sig, ctx) == want, name


def test_public_half_of_the_key_is_used_as_given(oe):
    seed, other = bytes([7]) * 57, bytes([8]) * 57
    wrong = M.public(other)
    sig = oe.ed448_sign(seed + wrong, b"message")
    assert sig == M.sign(seed, wrong, b"message")
    assert sig != oe.ed448_sign(oe.ed448_keygen(seed)[1], b"message")


def _edd3_reference(seed, msg):
    import oracle
    from cryptography.hazmat.primitives.asymmetric.ed448 import Ed448PrivateKey
    ex = hashlib.shake_256(seed).digest(89)
    dpk, dsk = oracle.mldsa_keygen(3, ex[:32])
    k = Ed448PrivateKey.from_private_bytes(ex[32:])
    pk, sk = dpk + k.public_key().public_bytes_raw(), dsk + ex[32:]
    return pk, sk, oracle.mldsa_sign(3, dsk, msg)[0] + k.sign(msg)


def test_eddilithium3_rebuilt_from_parts(oe):
    rng = random.Random(2)
    for n in (0, 1, 137, 500):
        seed = bytes(rng.randrange(256) for _ in range(57))
        msg = bytes(rng.randrange(256) for _ in range(n))
        pk, sk, sig = _edd3_reference(seed, msg)
        assert (len(pk), len(sk), len(sig)) == (2009, 4057, 3407)
        assert oe.eddilithium3_keygen(seed) == (pk, sk)
        assert oe.eddilithium3_sign(sk, msg) == sig
        assert oe.eddilithium3_verify(pk, msg, sig)
        for pos in (10, 3300, 3406):
            bad = bytearray(sig)
            bad[pos] ^= 1
            assert not oe.eddilithium3_verify(pk, msg, bytes(bad))
        assert not oe.eddilithium3_verify(pk, msg, sig[:-1])
