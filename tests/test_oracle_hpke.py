"""Oracle pins for HPKE's DHKEM(X25519, HKDF-SHA256) and DHKEM(X448, HKDF-SHA512): the RFC 9180 vectors of the
reference (hpke/testdata, every mode), and random seeds against an independent model built from OpenSSL's
X25519 / X448 and Python's hmac (tests/hpke_model.py), including the low-order failures."""
import hashlib
import random

import pytest

import hpke_model as M
from conftest import load_golden
from oracle import hpke as oh

IDS = [M.X25519_ID, M.X448_ID]


@pytest.fixture(scope="module")
def vectors():
    return load_golden("hpke_vectors.json.gz")["vectors"]


def _b(v, k):
    return bytes.fromhex(v[k])


def test_fixture_covers_both_ids_and_all_modes(vectors):
    assert len(vectors) == 64
    assert {(v["kem_id"], v["mode"]) for v in vectors} == {(i, m) for i in IDS for m in range(4)}


def test_oracle_reproduces_rfc9180_vectors(vectors):
    for v in vectors:
        kid, auth = v["kem_id"], v["mode"] in (2, 3)
        for who in "ERS" if auth else "ER":
            pk, sk = oh.keygen(kid, _b(v, "ikm" + who))
            assert (pk, sk) == (_b(v, f"pk{who}m"), _b(v, f"sk{who}m")), who
        skS = _b(v, "skSm") if auth else None
        pkS = _b(v, "pkSm") if auth else None
        enc, ss, rc = oh.encaps(kid, _b(v, "pkRm"), _b(v, "ikmE"), skS)
        assert (enc, ss, rc) == (_b(v, "enc"), _b(v, "shared_secret"), 0)
        assert oh.decaps(kid, _b(v, "skRm"), enc, pkS) == (_b(v, "shared_secret"), 0)


def test_model_reproduces_rfc9180_vectors(vectors):
    for v in vectors:
        m = M.KEMS[v["kem_id"]]
        if v["mode"] in (2, 3):
            enc, ss = m.auth_encaps(_b(v, "pkRm"), _b(v, "skSm"), _b(v, "ikmE"))
        else:
            enc, ss = m.encaps(_b(v, "pkRm"), _b(v, "ikmE"))
        assert (enc, ss) == (_b(v, "enc"), _b(v, "shared_secret"))


def test_hashes_against_hashlib():
    rng = random.Random(5)
    for n in list(range(0, 300)) + [1000]:
        m = bytes(rng.randrange(256) for _ in range(n))
        assert oh.sha256(m) == hashlib.sha256(m).digest()
        assert oh.sha512(m) == hashlib.sha512(m).digest()


@pytest.mark.parametrize("kid", IDS)
def test_oracle_matches_model_on_random_seeds(kid):
    m, n = M.KEMS[kid], M.KEMS[kid].n
    rng = random.Random(kid)
    rb = lambda: bytes(rng.randrange(256) for _ in range(n))  # noqa: E731
    for _ in range(40):
        pkR, skR = oh.keygen(kid, rb())
        pkS, skS = oh.keygen(kid, rb())
        seed = rb()
        sk, pk = m.derive(seed)
        assert oh.keygen(kid, seed) == (pk, sk)
        seed = rb()
        enc, ss, rc = oh.encaps(kid, pkR, seed)
        assert rc == 0 and (enc, ss) == m.encaps(pkR, seed)
        assert oh.decaps(kid, skR, enc) == (ss, 0) and m.decaps(skR, enc) == ss
        enc, ss, rc = oh.encaps(kid, pkR, seed, skS)
        assert rc == 0 and (enc, ss) == m.auth_encaps(pkR, skS, seed)
        assert oh.decaps(kid, skR, enc, pkS) == (ss, 0) and m.auth_decaps(skR, enc, pkS) == ss
        # a random private key that is not clamped is used as given (KeyGen clamps it)
        raw = rb()
        assert oh.decaps(kid, raw, enc)[0] == m.decaps(raw, enc)


@pytest.mark.parametrize("kid", IDS)
def test_low_order_shares_fail(kid):
    m, n = M.KEMS[kid], M.KEMS[kid].n
    pkR, skR = oh.keygen(kid, b"\x01" * n)
    pkS, skS = oh.keygen(kid, b"\x02" * n)
    seed = b"\x03" * n
    enc, _, _ = oh.encaps(kid, pkR, seed)
    for bad in M.low_order_points(kid):
        with pytest.raises(M.LowOrder):
            m.shared(skR, bad)
        assert oh.encaps(kid, bad, seed)[1:] == (bytes(m.nh), 1)          # pkR
        assert oh.encaps(kid, bad, seed, skS)[1:] == (bytes(m.nh), 1)     # pkR, auth
        assert oh.decaps(kid, skR, bad) == (bytes(m.nh), 1)               # enc
        assert oh.decaps(kid, skR, bad, pkS) == (bytes(m.nh), 1)          # enc, auth
        assert oh.decaps(kid, skR, enc, bad) == (bytes(m.nh), 1)          # pkS


def test_bit_255_of_x25519_keys_enters_kem_context():
    """Shared masks bit 255 of pkR, kem_context keeps the bytes as given: same dh, different ss."""
    m = M.KEMS[M.X25519_ID]
    pkR, skR = oh.keygen(M.X25519_ID, b"\x05" * 32)
    hi = pkR[:31] + bytes([pkR[31] | 0x80])
    seed = b"\x06" * 32
    enc, ss, rc = oh.encaps(M.X25519_ID, pkR, seed)
    enc2, ss2, rc2 = oh.encaps(M.X25519_ID, hi, seed)
    assert rc == rc2 == 0 and enc == enc2 and ss != ss2
    skE, _ = m.derive(seed)
    assert m.kdf(m.shared(skE, pkR), enc + hi) == ss2
    # and on the receiving side, an enc with bit 255 set
    enc_hi = enc[:31] + bytes([enc[31] | 0x80])
    assert oh.decaps(M.X25519_ID, skR, enc_hi)[0] == m.kdf(m.shared(skR, enc), enc_hi + pkR) != ss
