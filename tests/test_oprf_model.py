"""tests/oprf_model.py against the reference's fixtures: every NIST-suite RFC 9497 vector in all three modes (skSm and
pkSm from seed and keyInfo, EvaluationElement and Proof given r, Output, the client's Blind, proof check and Finalize),
the RFC 9380 hash_to_curve vectors with their u, Q0 and Q1, and the expand_message_xmd vectors."""
import pytest

import oprf_model as om
from conftest import load_golden

NIST = [v for v in load_golden("oprf_rfc9497.json.gz") if v["identifier"] in om.SUITES]


def test_fixture_covers_every_nist_suite_and_mode():
    assert sorted((v["identifier"], v["mode"]) for v in NIST) == sorted(
        (i, m) for i in om.SUITES for m in (0, 1, 2))


def _x(h):
    return bytes.fromhex(h)


@pytest.mark.parametrize("tv", NIST, ids=lambda v: f"{v['identifier']}-mode{v['mode']}")
def test_rfc9497_vectors(tv):
    s, mode = om.SUITES[tv["identifier"]], tv["mode"]
    assert _x(tv["groupDST"]) == b"HashToGroup-" + om.context(s, mode)
    sk, pk = om.derive_key(s, mode, _x(tv["seed"]), _x(tv["keyInfo"]))
    assert sk.hex() == tv["skSm"]
    if "pkSm" in tv:
        assert pk.hex() == tv["pkSm"]
    for v in tv["vectors"]:
        inputs = [_x(h) for h in v["Input"].split(",")]
        blinds = [int(h, 16) for h in v["Blind"].split(",")]
        blinded = [_x(h) for h in v["BlindedElement"].split(",")]
        info = _x(v.get("Info", ""))
        assert [om.blind(s, mode, i, b) for i, b in zip(inputs, blinds)] == blinded
        r = _x(v["Proof"]["r"]) if "Proof" in v else None
        ev, proof = om.evaluate(s, mode, sk, blinded, r, info)
        assert [e.hex() for e in ev] == v["EvaluationElement"].split(",")
        if mode == om.BASE:
            assert proof is None
        else:
            assert proof.hex() == v["Proof"]["proof"]
            assert om.client_verify(s, mode, pk, blinded, ev, proof, info)
            bad = bytes([proof[0] ^ 1]) + proof[1:]
            assert not om.client_verify(s, mode, pk, blinded, ev, bad, info)
        outs = v["Output"].split(",")
        for i, b, e, o in zip(inputs, blinds, ev, outs):
            assert om.finalize(s, mode, i, b, e, info).hex() == o
            assert om.full_evaluate(s, mode, sk, i, info).hex() == o


H2C = {"P256-SHA256": "h2c_P256_XMD-SHA-256_SSWU_RO_.json.gz", "P384-SHA384": "h2c_P384_XMD-SHA-384_SSWU_RO_.json.gz",
       "P521-SHA512": "h2c_P521_XMD-SHA-512_SSWU_RO_.json.gz"}


@pytest.mark.parametrize("ident", list(H2C))
def test_rfc9380_hash_to_curve(ident):
    s, f = om.SUITES[ident], load_golden(H2C[ident])
    assert int(f["L"], 16) == s.L and int(f["Z"], 16) == s.Z % s.p and int(f["field"]["p"], 16) == s.p
    for v in f["vectors"]:
        u, q0, q1, pt = om.hash_to_curve(s, v["msg"].encode(), f["dst"].encode())
        assert u == [int(x, 16) for x in v["u"]]
        for got, name in ((q0, "Q0"), (q1, "Q1"), (pt, "P")):
            assert got == (int(v[name]["x"], 16), int(v[name]["y"], 16)), name
            assert om.on_curve(s, got)


XMD = {"expand_message_xmd_SHA256_38.json.gz": om.hashlib.sha256, "expand_message_xmd_SHA256_256.json.gz": om.hashlib.sha256,
       "expand_message_xmd_SHA512_38.json.gz": om.hashlib.sha512}


@pytest.mark.parametrize("name", list(XMD))
def test_expand_message_xmd(name):
    f = load_golden(name)
    for v in f["tests"]:
        out = om.expand_message_xmd(XMD[name], v["msg"].encode(), f["DST"].encode(), int(v["len_in_bytes"], 16))
        assert out.hex() == v["uniform_bytes"]


@pytest.mark.parametrize("s", list(om.SUITES.values()), ids=list(om.SUITES))
def test_decompress_edges(s):
    g = om.compress(s, s.g)
    assert om.decompress(s, g) == s.g
    neg = bytes([g[0] ^ 1]) + g[1:]
    assert om.decompress(s, neg) == (s.g[0], s.p - s.g[1])
    assert om.decompress(s, b"\x04" + g[1:]) is None
    assert om.decompress(s, b"\x02" + om.i2osp(s.p, s.nbytes)) is None
    x = next(x for x in range(1, 100) if not om._is_square(s, (x ** 3 - 3 * x + s.b) % s.p))
    assert om.decompress(s, b"\x02" + om.i2osp(x, s.nbytes)) is None


@pytest.mark.parametrize("s", list(om.SUITES.values()), ids=list(om.SUITES))
def test_partial_key_with_t_zero_fails(s):
    info = b"t = 0"
    sk = om.i2osp(s.n - om.info_scalar(s, info), s.Ns)
    with pytest.raises(om.OprfError) as e:
        om.full_evaluate(s, om.PARTIAL, sk, b"x", info)
    assert e.value.status == 8


@pytest.mark.parametrize("mode", [om.BASE, om.VERIFIABLE, om.PARTIAL])
@pytest.mark.parametrize("s", list(om.SUITES.values()), ids=list(om.SUITES))
def test_grouped_evaluate_matches_evaluate(s, mode):
    """evaluate_grouped, which the large GPU batches are checked with, gives evaluate's elements, proof and errors
    byte for byte, at m from 1 to 40 with repeated elements (a weight sum that wraps mod n included)."""
    import random
    rng = random.Random(9497 + 10 * mode + s.bits)
    pool = [om.compress(s, om.mul(s, rng.randrange(1, s.n), s.g)) for _ in range(4)]
    info = b"grouped" if mode == om.PARTIAL else b""
    for m in (1, 2, 3, 7, 16, 40):
        sk = om.i2osp(rng.randrange(1, s.n), s.Ns)
        r = om.i2osp(rng.randrange(1, s.n), s.Ns)
        bl = [pool[0]] * m if m == 16 else [pool[rng.randrange(len(pool))] for _ in range(m)]
        assert om.evaluate_grouped(s, mode, sk, bl, r, info) == om.evaluate(s, mode, sk, bl, r, info), m
    # the same status bits on failing requests
    x = next(v for v in range(1, 200) if not om._is_square(s, (v ** 3 - 3 * v + s.b) % s.p))
    bad = [b"\x02" + om.i2osp(x, s.nbytes), b"\x04" + pool[0][1:]]
    t0 = om.i2osp(s.n - om.info_scalar(s, info), s.Ns) if mode == om.PARTIAL else bytes(s.Ns)
    one = om.i2osp(1, s.Ns)
    for sk, bl, r in ((bytes(s.Ns), pool[:2], one), (om.i2osp(s.n, s.Ns), pool[:2], one), (one, pool[:1] + bad, one),
                      (one, pool[:2], bytes(s.Ns)), (t0, pool[:2], one), (bytes(s.Ns), bad, bytes(s.Ns))):
        want = got = None
        try:
            want = om.evaluate(s, mode, sk, bl, r, info)
        except om.OprfError as e:
            want = e.status
        try:
            got = om.evaluate_grouped(s, mode, sk, bl, r, info)
        except om.OprfError as e:
            got = e.status
        assert got == want
