"""Oracle pins for DHKEM(P-256, HKDF-SHA256) (oracle/p256.c): the 32 RFC 9180 vectors of kem_id 0x10, OpenSSL's ECDH
and HPKE (cryptography) on random keys, its point decoder on invalid encodings, and the candidate-loop seed."""
import hashlib
import hmac
import random

import pytest

from conftest import load_golden

P = 2**256 - 2**224 + 2**192 + 2**96 - 1
N = 0xffffffff00000000ffffffffffffffffbce6faada7179e84f3b9cac2fc632551


@pytest.fixture(scope="module")
def op():
    from oracle import p256
    p256.build()
    return p256


def test_rfc9180_vectors(op):
    vs = load_golden("hpke_p256_vectors.json.gz")["vectors"]
    assert len(vs) == 32 and sorted({v["mode"] for v in vs}) == [0, 1, 2, 3]
    for v in vs:
        h = lambda k: bytes.fromhex(v[k])  # noqa: E731
        for who in "ERS" if v["mode"] in (2, 3) else "ER":
            assert op.keygen(h("ikm" + who))[:2] == (h(f"pk{who}m"), h(f"sk{who}m"))
        skS, pkS = (h("skSm"), h("pkSm")) if v["mode"] in (2, 3) else (None, None)
        assert op.encaps(h("pkRm"), h("ikmE"), skS) == (h("enc"), h("shared_secret"), 0)
        assert op.decaps(h("skRm"), h("enc"), pkS) == (h("shared_secret"), 0)


def test_candidate_loop_seed(op):
    fx = load_golden("hpke_p256_vectors.json.gz")["ctr_seeds"]
    assert fx
    for f in fx:
        seed = bytes.fromhex(f["ikm"])
        # the ctr = 0 candidate, computed here with hmac, is not below n
        sid = b"KEM\x00\x10"
        prk = hmac.new(bytes(32), b"HPKE-v1" + sid + b"dkp_prk" + seed, hashlib.sha256).digest()
        c0 = hmac.new(prk, b"\x00\x20HPKE-v1" + sid + b"candidate\x00\x01", hashlib.sha256).digest()
        assert int.from_bytes(c0, "big") >= N
        assert op.keygen(seed) == (bytes.fromhex(f["pk"]), bytes.fromhex(f["sk"]), f["ctr"])


def _ossl_pub(k):
    from cryptography.hazmat.primitives import serialization as ser
    return k.public_key().public_bytes(ser.Encoding.X962, ser.PublicFormat.UncompressedPoint)


def test_ecdh_against_openssl(op):
    from cryptography.hazmat.primitives.asymmetric import ec
    for _ in range(64):
        a, b = ec.generate_private_key(ec.SECP256R1()), ec.generate_private_key(ec.SECP256R1())
        ska = a.private_numbers().private_value.to_bytes(32, "big")
        assert op.ecdh(ska) == (_ossl_pub(a), 0)
        assert op.ecdh(ska, _ossl_pub(b)) == (a.exchange(ec.ECDH(), b.public_key()), 0)
    for k in (1, 2, N - 1, N - 2):
        want = _ossl_pub(ec.derive_private_key(k, ec.SECP256R1()))
        assert op.ecdh(k.to_bytes(32, "big")) == (want, 0)


def test_point_decoder_agrees_with_openssl(op):
    from cryptography.hazmat.primitives.asymmetric import ec
    g = _ossl_pub(ec.derive_private_key(1, ec.SECP256R1()))
    x, y = int.from_bytes(g[1:33], "big"), int.from_bytes(g[33:], "big")
    cands = [g, b"\x04" + bytes(64), b"\x04" + x.to_bytes(32, "big") + ((y + 1) % P).to_bytes(32, "big"),
             b"\x04" + P.to_bytes(32, "big") + y.to_bytes(32, "big"), b"\x04" + x.to_bytes(32, "big") + P.to_bytes(32, "big"),
             b"\x04" + x.to_bytes(32, "big") + (P - y).to_bytes(32, "big"), b"\x04" + b"\xff" * 64]
    cands += [bytes([pre]) + g[1:] for pre in (0x00, 0x02, 0x03, 0x05, 0x06, 0x07)]
    rng = random.Random(5)
    cands += [b"\x04" + bytes(rng.randrange(256) for _ in range(64)) for _ in range(20)]
    for c in cands:
        try:
            ec.EllipticCurvePublicKey.from_encoded_point(ec.SECP256R1(), c)
            want = True
        except ValueError:
            want = False
        assert op.point_ok(c) == want, c.hex()
    for k, ok in ((0, False), (1, True), (N - 1, True), (N, False), (2**256 - 1, False)):
        assert op.scalar_ok(k.to_bytes(32, "big")) == ok
    # invalid inputs: the status bits and all-zero outputs
    assert op.ecdh(N.to_bytes(32, "big")) == (bytes(65), 2)
    assert op.ecdh((5).to_bytes(32, "big"), b"\x02" + g[1:]) == (bytes(32), 1)
    assert op.encaps(b"\x05" + g[1:], bytes(32))[1:] == (bytes(32), 1)
    assert op.decaps(bytes(32), g)[1] == 2


def test_hpke_against_openssl(op):
    """OpenSSL's HPKE seals to a key, the oracle decapsulates, and the RFC 9180 key schedule (written out here) opens."""
    from cryptography.hazmat.primitives import hpke
    from cryptography.hazmat.primitives.asymmetric import ec
    from cryptography.hazmat.primitives.ciphers.aead import AESGCM
    suite = hpke.Suite(hpke.KEM.P256, hpke.KDF.HKDF_SHA256, hpke.AEAD.AES_128_GCM)
    sid = b"HPKE" + (0x10).to_bytes(2, "big") + (1).to_bytes(2, "big") + (1).to_bytes(2, "big")
    ext = lambda salt, lab, ikm: hmac.new(salt or bytes(32), b"HPKE-v1" + sid + lab + ikm, hashlib.sha256).digest()  # noqa: E731
    exp = lambda prk, lab, inf, L: hmac.new(prk, L.to_bytes(2, "big") + b"HPKE-v1" + sid + lab + inf + b"\x01",  # noqa: E731
                                            hashlib.sha256).digest()[:L]
    ctx = b"\x00" + ext(b"", b"psk_id_hash", b"") + ext(b"", b"info_hash", b"")
    for i in range(16):
        k = ec.generate_private_key(ec.SECP256R1())
        ct = suite.encrypt(b"msg %d" % i, k.public_key())
        ss, st = op.decaps(k.private_numbers().private_value.to_bytes(32, "big"), ct[:65])
        assert st == 0
        secret = ext(ss, b"secret", b"")
        assert AESGCM(exp(secret, b"key", ctx, 16)).decrypt(exp(secret, b"base_nonce", ctx, 12), ct[65:], b"") == b"msg %d" % i
