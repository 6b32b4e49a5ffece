"""CPU-only: tests/brsa_model.py against the four RFC 9474 vectors (every field: the blinded message from input_msg,
salt and inv, then blind_sig and sig) and against OpenSSL through the cryptography package (each final signature
verifies as RSA-PSS-SHA-384 with salt length 48 or 0, and OpenSSL's own PSS signatures verify under the model)."""
import pytest

import brsa_model as bm

crypto = pytest.importorskip("cryptography")
from cryptography.hazmat.primitives import hashes  # noqa: E402
from cryptography.hazmat.primitives.asymmetric import padding, rsa  # noqa: E402


def _x(h):
    return bytes.fromhex(h)


def _openssl_public(k):
    return rsa.RSAPublicNumbers(k.e, k.n).public_key()


def _openssl_private(k):
    dp, dq, qinv = k.crt()
    return rsa.RSAPrivateNumbers(k.p, k.q, k.d, dp, dq, qinv, rsa.RSAPublicNumbers(k.e, k.n)).private_key()


@pytest.mark.parametrize("variant", range(4), ids=[v[0] for v in bm.VARIANTS])
def test_rfc9474_vector(variant):
    v = bm.rfc_vectors()[variant]
    name, slen, plen = bm.VARIANTS[variant]
    assert v["name"].upper() == name.upper() and int(v["sLen"], 16) == slen
    k = bm.rfc_key()
    prepared = bm.prepare(variant, _x(v["msg"]), _x(v["msg_prefix"]) if plen else b"")
    assert prepared.hex() == v["input_msg"]
    inv = int(v["inv"], 16)
    blinded, inv2 = bm.blind(k, variant, prepared, _x(v["salt"]) if slen else b"", pow(inv, -1, k.n))
    assert blinded.hex() == v["blinded_msg"] and inv2 == inv
    st, bs = bm.blind_sign(k, blinded)
    assert st == 0 and bs.hex() == v["blind_sig"]
    sig = bm.finalize(k, variant, prepared, bs, inv)
    assert sig.hex() == v["sig"]
    _openssl_public(k).verify(sig, prepared, padding.PSS(padding.MGF1(hashes.SHA384()), slen), hashes.SHA384())


@pytest.mark.parametrize("name", ["rsa2048", "rsa3072", "rsa3073", "rsa2048e3", "rsa2048u", "rsa3000u"])
def test_fixture_keys_against_openssl(name):
    k = bm.all_keys()[name]
    assert k.n == k.p * k.q and pow(pow(7, k.e, k.n), k.d, k.n) == 7
    sk = _openssl_private(k)
    for slen in (48, 0):
        msg = b"fixture key " + name.encode()
        sig = sk.sign(msg, padding.PSS(padding.MGF1(hashes.SHA384()), slen), hashes.SHA384())
        assert bm.verify_status(k, slen, msg, sig) == 0
        # a PSS signature with the other salt length fails
        assert bm.verify_status(k, 48 - slen, msg, sig) == 2


def test_blind_sign_edges():
    k = bm.pem_key()
    n = k.n
    assert bm.blind_sign(k, bm.i2osp(0, k.klen)) == (0, bytes(k.klen))
    assert bm.blind_sign(k, bm.i2osp(n, k.klen))[0] == 2
    assert bm.blind_sign(k, bm.i2osp(n + 1, k.klen))[0] == 1
    assert bm.blind_sign(k, bm.i2osp(n - 1, k.klen)) == (0, bm.i2osp(n - 1, k.klen))  # (-1)^d = -1 for odd d
