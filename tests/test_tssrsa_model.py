"""CPU-only: tests/tssrsa_model.py and the host parts of circl_b200.tssrsa (Deal, the encodings, PadHash and the
parameter checks of CombineSignShares) against the data of the reference's tests (tests/golden/tssrsa_reference.json.gz),
and the model's combined signatures against OpenSSL under the full key: PKCS #1 v1.5 signatures byte-equal to OpenSSL's
(an e-th root mod N is unique), PSS signatures verifying."""
import random

import pytest

import brsa_model as bm
import tssrsa_model as tm

REF = tm.reference_data()


class _Bytes:
    def __init__(self, b):
        self.b = bytes(b)

    def read(self, n):
        out, self.b = self.b[:n], self.b[n:]
        return out


class _Stream:
    def __init__(self, rng):
        self.rng = rng

    def read(self, n):
        return self.rng.randbytes(n)


class _Pub:
    def __init__(self, n, e):
        self.N, self.E = n, e


def test_deal_sign_delta_lambda():
    from circl_b200 import tssrsa
    d = REF["deal"]
    assert tm.deal(_Bytes(d["stream"]), d["players"], d["threshold"], d["p"], d["q"], d["e"]) == d["si"]
    key = type("K", (), {"E": d["e"], "Primes": [d["p"], d["q"]]})
    shares = tssrsa.Deal(_Bytes(d["stream"]), d["players"], d["threshold"], key, False)
    assert [s.si for s in shares] == d["si"] and [s.Index for s in shares] == [1, 2, 3]
    assert all(s.twoDeltaSi is None for s in shares)
    cached = tssrsa.Deal(_Bytes(d["stream"]), d["players"], d["threshold"], key, True)
    assert [s.twoDeltaSi for s in cached] == [12 * v for v in d["si"]]
    s = REF["sign"]
    assert tm.sign_share(s["n"], 2 * tm.delta(s["players"]) * s["si"], s["x"]) == s["xi"]
    for l, want in REF["delta"]:
        assert tm.delta(l) == want
    for c in REF["lambda"]:
        assert tm.compute_lambda(tm.delta(c["l"]), c["S"], c["i"], c["j"], c["l"]) == int(c["want"])
    ci = REF["check_indices"]
    for want in (True, False):
        for i, j in ci["true" if want else "false"]:
            assert tm.check_indices(i, j, ci["l"], ci["S"]) == want, (i, j)


def test_encodings():
    from circl_b200 import tssrsa
    for c in REF["keyshare_ok"]:
        a = tssrsa.KeyShare(c["si"], c["index"], c["players"], c["threshold"], c["twoDeltaSi"])
        b = tssrsa.KeyShare()
        b.UnmarshalBinary(a.MarshalBinary())
        assert vars(a) == vars(b)
    for h in REF["keyshare_bad"]:
        with pytest.raises(ValueError):
            tssrsa.KeyShare().UnmarshalBinary(bytes.fromhex(h))
    for c in REF["signshare_ok"]:
        a = tssrsa.SignShare(c["xi"], c["index"], c["players"], c["threshold"])
        b = tssrsa.SignShare()
        b.UnmarshalBinary(a.MarshalBinary())
        assert vars(a) == vars(b)
    for h in REF["signshare_bad"]:
        with pytest.raises(ValueError):
            tssrsa.SignShare().UnmarshalBinary(bytes.fromhex(h))
    for n in REF["keyshare_wrap"]:
        data = bytearray(8 + n)
        data[6:8] = n.to_bytes(2, "big")
        data[8] = 1
        with pytest.raises(ValueError):
            tssrsa.KeyShare().UnmarshalBinary(bytes(data))
    for n in REF["signshare_wrap"]:
        data = bytearray(8 + n)
        data[6:8] = n.to_bytes(2, "big")
        data[8] = 1
        s = tssrsa.SignShare()
        s.UnmarshalBinary(bytes(data))
        assert s.xi == 1 << (8 * (n - 1))
    # the exact layout: | Players | Threshold | Index | siLen | si | nil flag | twoDeltaSiLen | twoDeltaSi |
    assert tssrsa.KeyShare(10, 30, 2, 10, 20).MarshalBinary().hex() == "0002000a001e00010a01000114"
    assert tssrsa.KeyShare(0, 0, 0, 0, None).MarshalBinary().hex() == "000000000000000100000000"
    assert tssrsa.SignShare(0, 0, 0, 0).MarshalBinary().hex() == "000000000000000100"
    with pytest.raises(ValueError, match="Index is too big"):
        tssrsa.SignShare(1, 1 << 16, 3, 2).MarshalBinary()


def test_combine_parameter_errors_in_the_reference_order():
    from circl_b200 import tssrsa
    u = REF["untrusted"]
    share = tssrsa.SignShare()
    share.UnmarshalBinary(bytes.fromhex(u["share"]))
    assert (share.Players, share.Threshold, share.Index, share.xi) == (65535, 1, 1, 2)
    with pytest.raises(ValueError) as ei:
        tssrsa.CombineSignShares(_Pub(u["n"], u["e"]), u["players"], u["threshold"], [share], bytes.fromhex(u["msg"]))
    assert str(ei.value) == u["error"]
    pub = _Pub(3233, 17)
    ok = [tssrsa.SignShare(2, i, 3, 2) for i in (1, 2)]
    for args, msg in (((1, 1, ok), "Players \\(l\\) invalid"), ((3, 0, ok), "Threshold \\(k\\) invalid"),
                      ((3, 2, []), "no shares provided"),
                      ((3, 2, [tssrsa.SignShare(2, 1, 3, 3)]), "share threshold did not match"),
                      ((3, 2, ok[:1]), "insufficient shares")):
        with pytest.raises(ValueError, match=msg):
            tssrsa.CombineSignShares(pub, *args, b"\x01")
    with pytest.raises(tssrsa.ErrInvalidCalc):
        tssrsa.CombineSignShares(pub, 3, 2, [tssrsa.SignShare(2, 0, 3, 2)] + ok, b"\x01")


@pytest.mark.parametrize("name,players,threshold", [("rsa2048", 3, 2), ("rsa2048", 5, 3), ("rsa3072", 4, 4)])
def test_model_signatures_match_openssl(name, players, threshold):
    from cryptography.hazmat.primitives import hashes
    from cryptography.hazmat.primitives.asymmetric import padding, rsa
    from circl_b200 import tssrsa
    k = bm.all_keys()[name]
    osk = rsa.RSAPrivateNumbers(k.p, k.q, k.d, k.d % (k.p - 1), k.d % (k.q - 1), pow(k.q, -1, k.p),
                                rsa.RSAPublicNumbers(k.e, k.n)).private_key()
    rng = random.Random(name + str(players))
    si = tm.deal(_Stream(rng), players, threshold, k.p, k.q, k.e)
    pub = _Pub(k.n, k.e)
    for h, ch in (("sha256", hashes.SHA256()), ("sha384", hashes.SHA384())):
        for pss in (False, True):
            m = rng.randbytes(40)
            padder = tssrsa.PSSPadder(_Stream(rng)) if pss else tssrsa.PKCS1v15Padder()
            x = int.from_bytes(tssrsa.PadHash(padder, h, pub, m), "big")
            S = sorted(rng.sample(range(1, players + 1), threshold))
            xi = [tm.sign_share(k.n, 2 * tm.delta(players) * si[j - 1], x) for j in S]
            st, y = tm.combine(k.n, k.e, players, S, xi, x)
            assert st == 0
            sig = y.to_bytes(k.klen, "big")
            if pss:
                osk.public_key().verify(sig, m, padding.PSS(padding.MGF1(ch), padding.PSS.AUTO), ch)
            else:
                assert sig == osk.sign(m, padding.PKCS1v15(), ch)


def test_batch_indices_outside_16_bits_are_refused():
    import numpy as np
    from circl_b200 import tssrsa
    k = bm.all_keys()["rsa2048"]
    pub, kl = _Pub(k.n, k.e), k.klen
    xi, msgs = np.zeros((1, 2 * kl), np.uint8), np.zeros((1, kl), np.uint8)
    for bad in ([[1, 65536]], [[1, 65537]], [[-1, 2]]):
        with pytest.raises(ValueError, match="0 .. 65535"):
            tssrsa.CombineSignSharesBatch(pub, 3, 2, np.array(bad, np.int64), xi, msgs)
    with pytest.raises(ValueError, match="integers"):
        tssrsa.CombineSignSharesBatch(pub, 3, 2, np.array([[1.0, 2.0]]), xi, msgs)
