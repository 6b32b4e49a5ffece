"""Oracle pins for DHKEM(P-384, HKDF-SHA384) and DHKEM(P-521, HKDF-SHA512) (oracle/nistp.c): the 32 RFC 9180 vectors of
kem_id 0x12, the hashlib / OpenSSL model of tests/nistp_model.py on both curves, OpenSSL's ECDH and point decoder, its
SHA-384, and OpenSSL's HPKE (cryptography) in both directions."""
import hashlib
import os
import random

import pytest

from conftest import load_golden
from nistp_model import CURVES
import nistp_model as model


@pytest.fixture(scope="module")
def op():
    from oracle import nistp
    nistp.build()
    return nistp


def test_rfc9180_vectors(op):
    vs = load_golden("hpke_p521_vectors.json.gz")["vectors"]
    assert len(vs) == 32 and sorted({v["mode"] for v in vs}) == [0, 1, 2, 3]
    for v in vs:
        h = lambda k: bytes.fromhex(v[k])  # noqa: E731
        for who in "ERS" if v["mode"] in (2, 3) else "ER":
            assert op.keygen(521, h("ikm" + who))[:2] == (h(f"pk{who}m"), h(f"sk{who}m"))
            assert model.derive_key_pair(CURVES[521], h("ikm" + who)) == (h(f"pk{who}m"), h(f"sk{who}m"))
        skS, pkS = (h("skSm"), h("pkSm")) if v["mode"] in (2, 3) else (None, None)
        assert op.encaps(521, h("pkRm"), h("ikmE"), skS) == (h("enc"), h("shared_secret"), 0)
        assert op.decaps(521, h("skRm"), h("enc"), pkS) == (h("shared_secret"), 0)


@pytest.mark.parametrize("bits", [384, 521])
def test_model(op, bits):
    c = CURVES[bits]
    rng = random.Random(bits)
    for _ in range(8):
        seeds = [bytes(rng.randrange(256) for _ in range(c.nbytes)) for _ in range(3)]
        pk, sk, _ = op.keygen(bits, seeds[0])
        pk2, sk2, _ = op.keygen(bits, seeds[1])
        assert (pk, sk) == model.derive_key_pair(c, seeds[0])
        for skS, pkS in ((None, None), (sk2, pk2)):
            enc, ss, st = op.encaps(bits, pk, seeds[2], skS)
            assert st == 0 and (enc, ss) == model.encaps(c, pk, seeds[2], skS)
            assert op.decaps(bits, sk, enc, pkS) == (ss, 0)


def test_sha384(op):
    for n in (0, 1, 111, 112, 127, 128, 239, 240, 1000):
        m = os.urandom(n)
        assert op.sha384(m) == hashlib.sha384(m).digest()


def _ossl_pub(k):
    from cryptography.hazmat.primitives import serialization as ser
    return k.public_key().public_bytes(ser.Encoding.X962, ser.PublicFormat.UncompressedPoint)


@pytest.mark.parametrize("bits", [384, 521])
def test_ecdh_and_point_decoder_against_openssl(op, bits):
    from cryptography.hazmat.primitives.asymmetric import ec
    c = CURVES[bits]
    nb, P, N = c.nbytes, c.p, c.n
    for _ in range(16):
        a, b = ec.generate_private_key(c.ossl()), ec.generate_private_key(c.ossl())
        ska = a.private_numbers().private_value.to_bytes(nb, "big")
        assert op.ecdh(bits, ska) == (_ossl_pub(a), 0)
        assert op.ecdh(bits, ska, _ossl_pub(b)) == (a.exchange(ec.ECDH(), b.public_key()), 0)
    for k in (1, 2, N - 1, N - 2):
        assert op.ecdh(bits, k.to_bytes(nb, "big")) == (_ossl_pub(ec.derive_private_key(k, c.ossl())), 0)
    g = _ossl_pub(ec.derive_private_key(1, c.ossl()))
    x, y = c.g
    cands = [g, b"\x04" + bytes(2 * nb), b"\x04" + x.to_bytes(nb, "big") + ((y + 1) % P).to_bytes(nb, "big"),
             b"\x04" + P.to_bytes(nb, "big") + y.to_bytes(nb, "big"), b"\x04" + x.to_bytes(nb, "big") + P.to_bytes(nb, "big"),
             b"\x04" + x.to_bytes(nb, "big") + (P - y).to_bytes(nb, "big"), b"\x04" + b"\xff" * (2 * nb)]
    cands += [bytes([pre]) + g[1:] for pre in (0x00, 0x02, 0x03, 0x05, 0x06, 0x07)]
    rng = random.Random(5)
    cands += [b"\x04" + bytes(rng.randrange(256) for _ in range(2 * nb)) for _ in range(10)]
    for cand in cands:
        try:
            ec.EllipticCurvePublicKey.from_encoded_point(c.ossl(), cand)
            want = True
        except ValueError:
            want = False
        assert op.point_ok(bits, cand) == want, cand.hex()
    for k, ok in ((0, False), (1, True), (N - 1, True), (N, False), (2**(8 * nb) - 1, False)):
        assert op.scalar_ok(bits, k.to_bytes(nb, "big")) == ok
    assert op.ecdh(bits, N.to_bytes(nb, "big")) == (bytes(c.npk), 2)
    assert op.ecdh(bits, (5).to_bytes(nb, "big"), b"\x02" + g[1:]) == (bytes(nb), 1)
    assert op.encaps(bits, b"\x05" + g[1:], bytes(nb))[1:] == (bytes(c.nss), 1)
    assert op.decaps(bits, bytes(nb), g)[1] == 2


@pytest.mark.parametrize("bits", [384, 521])
def test_hpke_against_openssl(op, bits):
    """Both directions: OpenSSL's HPKE seals to a key and the oracle's Decap gives the secret that opens it; the
    oracle's Encap to an OpenSSL key gives a secret whose sealed message OpenSSL opens.  The RFC 9180 key schedule
    around the KEM is tests/nistp_model.py's."""
    from cryptography.hazmat.primitives import hpke
    from cryptography.hazmat.primitives import serialization as ser
    from cryptography.hazmat.primitives.asymmetric import ec
    c = CURVES[bits]
    kdf = hpke.KDF.HKDF_SHA384 if bits == 384 else hpke.KDF.HKDF_SHA512
    suite = hpke.Suite(hpke.KEM.P384 if bits == 384 else hpke.KEM.P521, kdf, hpke.AEAD.AES_256_GCM)
    info = b"oracle interop"
    for i in range(4):
        k = ec.generate_private_key(c.ossl())
        sk = k.private_numbers().private_value.to_bytes(c.nbytes, "big")
        ct = suite.encrypt(b"msg %d" % i, k.public_key(), info=info)
        ss, st = op.decaps(bits, sk, ct[:c.npk])
        assert st == 0
        aead, nonce = model.schedule(c, ss, info)
        assert aead.decrypt(nonce, ct[c.npk:], b"") == b"msg %d" % i
        pk = k.public_key().public_bytes(ser.Encoding.X962, ser.PublicFormat.UncompressedPoint)
        enc, ss, st = op.encaps(bits, pk, os.urandom(c.nbytes))
        assert st == 0
        aead, nonce = model.schedule(c, ss, info)
        sealed = enc + aead.encrypt(nonce, b"back %d" % i, b"")
        assert suite.decrypt(sealed, k, info=info) == b"back %d" % i
