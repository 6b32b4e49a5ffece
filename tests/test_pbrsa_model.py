"""CPU-only: tests/pbrsa_model.py against the cryptography package (its HKDF, and OpenSSL's RSA-PSS-SHA-384 verify of
every final signature under (N, e') for moduli up to 3072 bits, above which OpenSSL caps public exponents at 64 bits),
and the model's client and signer round trip on every fixture key."""
import random

import pytest

import brsa_model as bm
import pbrsa_model as pm

crypto = pytest.importorskip("cryptography")
from cryptography.hazmat.primitives import hashes  # noqa: E402
from cryptography.hazmat.primitives.asymmetric import padding, rsa  # noqa: E402
from cryptography.hazmat.primitives.kdf.hkdf import HKDF  # noqa: E402

KEYS = ["strong2048", "safe3072", "safe4096", "safe2050", "safe2052", "safe3073", "safe2048u"]
METAS = [b"", b"m", b"metadata", bytes(range(256)) * 4]


def test_fixture_keys_are_safe_prime_keys():
    ks = pm.keys()
    assert sorted(ks) == sorted(KEYS)
    bits = {name: k.n.bit_length() for name, k in ks.items()}
    assert bits == {"strong2048": 2048, "safe3072": 3072, "safe4096": 4096, "safe2050": 2050, "safe2052": 2052,
                    "safe3073": 3073, "safe2048u": 2048}
    for k in ks.values():
        assert k.n == k.p * k.q and k.p % 4 == 3 and k.q % 4 == 3
        assert pow(pow(7, k.e, k.n), k.d, k.n) == 7
    u = ks["safe2048u"]
    assert sorted((u.p.bit_length(), u.q.bit_length())) == [960, 1088]
    # e' (1022 bits) exceeds q' of the 960-bit prime: the library reduces it
    assert pm.derive_public_key(u.n, b"") > min(u.p, u.q) // 2


@pytest.mark.parametrize("length", [1, 48, 96, 129, 200, 280])
def test_hkdf_matches_cryptography(length):
    rng = random.Random(length)
    salt, ikm, info = rng.randbytes(256), rng.randbytes(length), b"PBRSA"
    want = HKDF(hashes.SHA384(), length, salt, info).derive(ikm)
    assert pm.hkdf(salt, ikm, info, length) == want


@pytest.mark.parametrize("name", KEYS)
def test_derived_exponent_bits(name):
    k = pm.keys()[name]
    lam = k.n.bit_length() // 2
    for meta in METAS:
        e = pm.derive_public_key(k.n, meta)
        assert e & 1 and e < 1 << min(lam - 2, 8 * (lam // 8))
        assert e.bit_length() > lam - 16  # the top bytes are not all zero (overwhelmingly)


@pytest.mark.parametrize("name", KEYS)
def test_round_trip_and_openssl(name):
    k = pm.keys()[name]
    rng = random.Random(name)
    for meta in METAS:
        msg = rng.randbytes(rng.randrange(0, 200))
        sig = pm.sign(k, msg, meta, rng)
        assert pm.verify_status(k, msg, meta, sig) == 0
        assert pm.verify_status(k, msg, meta + b"x", sig) == 2
        assert pm.verify_status(k, msg + b"x", meta, sig) == 2
        if k.n.bit_length() <= 3072:
            e = pm.derive_public_key(k.n, meta)
            rsa.RSAPublicNumbers(e, k.n).public_key().verify(sig, pm.frame(msg, meta),
                                                             padding.PSS(padding.MGF1(hashes.SHA384()), 48),
                                                             hashes.SHA384())


def test_crt_route_and_edges():
    k = pm.keys()["strong2048"]
    qinv = pow(k.q, -1, k.p)
    rng = random.Random(7)
    for meta in METAS:
        c = bm.i2osp(rng.randrange(k.n), k.klen)
        assert pm.blind_sign(k, c, meta, qinv) == pm.blind_sign(k, c, meta)
        assert pm.blind_sign(k, c, meta, qinv + 1)[0] == 2
    assert pm.blind_sign(k, bm.i2osp(0, k.klen), b"") == (0, bytes(k.klen))
    assert pm.blind_sign(k, bm.i2osp(k.n, k.klen), b"")[0] == 2
    assert pm.blind_sign(k, bm.i2osp(k.n + 1, k.klen), b"")[0] == 1
