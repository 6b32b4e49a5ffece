"""GPU parity for P-384 / P-521 and HPKE's DHKEM(P-384, HKDF-SHA384) / DHKEM(P-521, HKDF-SHA512), each test on both
curves: the RFC 9180 vectors of kem_id 0x12 through the C ABI, the oracle on 2^12 random operations with per-op and
shared keys in every position, raw ECDH against OpenSSL (cryptography) at the edges of the scalar range, invalid keys
inside valid batches (host arrays, the C ABI and CUDA tensors), invalid shared keys, UnmarshalBinary* validation,
OpenSSL's HPKE in both directions, device rows at odd bytes, and host batches over two GPUs.  P-384 has no RFC vectors;
besides the oracle it is pinned against tests/nistp_model.py (hashlib / hmac and OpenSSL's ECDH)."""
import concurrent.futures as cf
import importlib

import numpy as np
import pytest

from conftest import load_golden
from nistp_model import CURVES
import nistp_model as model

pytestmark = pytest.mark.gpu

NAMES = {384: "HPKE_KEM_P384_HKDF_SHA384", 521: "HPKE_KEM_P521_HKDF_SHA512"}


@pytest.fixture(scope="module")
def cb():
    import circl_b200
    circl_b200.init(0)
    yield circl_b200
    circl_b200.shutdown()


@pytest.fixture(params=[384, 521], ids=["p384", "p521"])
def bits(request, cb):
    return request.param


def _mod(bits):
    return importlib.import_module(f"circl_b200.p{bits}")


def _scheme(bits):
    return _mod(bits).ByName(NAMES[bits])


def _rows(bs):
    return np.stack([np.frombuffer(bytes(b), dtype=np.uint8) for b in bs])


def _rand(n, w, seed):
    return np.random.default_rng(seed).integers(0, 256, size=(n, w), dtype=np.uint8)


def _pmap(fn, *cols):
    """fn over rows, in threads (the oracle's ctypes calls release the GIL)."""
    with cf.ThreadPoolExecutor(16) as ex:
        return list(ex.map(fn, *cols))


def _keys(bits, n, seed):
    return _scheme(bits).DeriveKeyPairBatch(_rand(n, CURVES[bits].nbytes, seed))


def test_rfc9180_vectors_through_the_c_abi(cb):
    s = _scheme(521)
    mine = load_golden("hpke_p521_vectors.json.gz")["vectors"]
    assert len(mine) == 32 and all(v["kem_id"] == 0x12 for v in mine)
    b = lambda vs, k: _rows([bytes.fromhex(v[k]) for v in vs])  # noqa: E731
    for who in "ER":
        pk, sk = s.DeriveKeyPairBatch(b(mine, "ikm" + who))
        assert np.array_equal(pk, b(mine, f"pk{who}m")) and np.array_equal(sk, b(mine, f"sk{who}m"))
    auth = [v for v in mine if v["mode"] in (2, 3)]
    base = [v for v in mine if v["mode"] in (0, 1)]
    pk, sk = s.DeriveKeyPairBatch(b(auth, "ikmS"))
    assert np.array_equal(pk, b(auth, "pkSm")) and np.array_equal(sk, b(auth, "skSm"))
    enc, ss = s.EncapsulateBatch(b(base, "pkRm"), b(base, "ikmE"))
    assert np.array_equal(enc, b(base, "enc")) and np.array_equal(ss, b(base, "shared_secret"))
    assert np.array_equal(s.DecapsulateBatch(b(base, "skRm"), b(base, "enc")), b(base, "shared_secret"))
    enc, ss = s.AuthEncapsulateBatch(b(auth, "pkRm"), b(auth, "skSm"), b(auth, "ikmE"))
    assert np.array_equal(enc, b(auth, "enc")) and np.array_equal(ss, b(auth, "shared_secret"))
    assert np.array_equal(s.AuthDecapsulateBatch(b(auth, "skRm"), b(auth, "enc"), b(auth, "pkSm")),
                          b(auth, "shared_secret"))
    v = auth[0]
    h = lambda k: bytes.fromhex(v[k])  # noqa: E731
    pkR, skR = s.DeriveKeyPair(h("ikmR"))
    assert (pkR.MarshalBinary(), skR.MarshalBinary()) == (h("pkRm"), h("skRm"))
    assert skR.Public().MarshalBinary() == h("pkRm")
    pkS, skS = s.UnmarshalBinaryPublicKey(h("pkSm")), s.UnmarshalBinaryPrivateKey(h("skSm"))
    assert s.AuthEncapsulateDeterministically(pkR, skS, h("ikmE")) == (h("enc"), h("shared_secret"))
    assert s.AuthDecapsulate(skR, h("enc"), pkS) == h("shared_secret")


def test_model_parity(bits):
    """DeriveKeyPair, AuthEncap and AuthDecap against the hashlib / OpenSSL model (the only pin of P-384 besides the
    oracle)."""
    c, s = CURVES[bits], _scheme(bits)
    n = 64
    seeds = _rand(n, c.nbytes, 61)
    pk, sk = s.DeriveKeyPairBatch(seeds)
    assert [(a.tobytes(), b.tobytes()) for a, b in zip(pk, sk)] == _pmap(lambda a: model.derive_key_pair(c, a.tobytes()),
                                                                         seeds)
    es = _rand(n, c.nbytes, 62)
    skS = np.roll(sk, 1, axis=0)
    enc, ss = s.AuthEncapsulateBatch(pk, skS, es)
    want = _pmap(lambda a, b, d: model.encaps(c, a.tobytes(), b.tobytes(), d.tobytes()), pk, es, skS)
    assert [(e.tobytes(), x.tobytes()) for e, x in zip(enc, ss)] == want
    pkS = np.roll(pk, 1, axis=0)
    assert [x.tobytes() for x in s.AuthDecapsulateBatch(sk, enc, pkS)] == [w[1] for w in want]


@pytest.mark.parametrize("shared", ["none", "R", "S", "RS"])
def test_oracle_parity_auth(bits, shared):
    """2^12 AuthEncap / AuthDecap with pkR / skR and skS / pkS per op or shared by the batch."""
    from oracle import nistp as op
    s = _scheme(bits)
    n = 1 << 12
    pkR, skR = _keys(bits, n, 1)
    pkS, skS = _keys(bits, n, 2)
    es = _rand(n, CURVES[bits].nbytes, 3)
    if "R" in shared:
        pkR_arg, skR_arg = s.UnmarshalBinaryPublicKey(pkR[0].tobytes()), s.UnmarshalBinaryPrivateKey(skR[0].tobytes())
        pkR, skR = pkR[:1].repeat(n, 0), skR[:1].repeat(n, 0)
    else:
        pkR_arg, skR_arg = pkR, skR
    if "S" in shared:
        pkS_arg, skS_arg = s.UnmarshalBinaryPublicKey(pkS[0].tobytes()), s.UnmarshalBinaryPrivateKey(skS[0].tobytes())
        pkS, skS = pkS[:1].repeat(n, 0), skS[:1].repeat(n, 0)
    else:
        pkS_arg, skS_arg = pkS, skS
    enc, ss = s.AuthEncapsulateBatch(pkR_arg, skS_arg, es)
    want = _pmap(lambda a, b, c: op.encaps(bits, a.tobytes(), b.tobytes(), c.tobytes()), pkR, es, skS)
    assert [(e.tobytes(), x.tobytes(), 0) for e, x in zip(enc, ss)] == want
    assert np.array_equal(s.AuthDecapsulateBatch(skR_arg, enc, pkS_arg), ss)


@pytest.mark.parametrize("shared", [False, True])
def test_oracle_parity_base(bits, shared):
    from oracle import nistp as op
    s = _scheme(bits)
    n = 1 << 12
    seeds = _rand(n, CURVES[bits].nbytes, 4)
    pk, sk = s.DeriveKeyPairBatch(seeds)
    got = _pmap(lambda a: op.keygen(bits, a.tobytes())[:2], seeds)
    assert [(a.tobytes(), b.tobytes()) for a, b in zip(pk, sk)] == got
    es = _rand(n, CURVES[bits].nbytes, 5)
    if shared:
        pk_arg, sk_arg = s.UnmarshalBinaryPublicKey(pk[0].tobytes()), s.UnmarshalBinaryPrivateKey(sk[0].tobytes())
        pk, sk = pk[:1].repeat(n, 0), sk[:1].repeat(n, 0)
    else:
        pk_arg, sk_arg = pk, sk
    enc, ss = s.EncapsulateBatch(pk_arg, es)
    want = _pmap(lambda a, b: op.encaps(bits, a.tobytes(), b.tobytes()), pk, es)
    assert [(e.tobytes(), x.tobytes(), 0) for e, x in zip(enc, ss)] == want
    got = s.DecapsulateBatch(sk_arg, enc)
    assert [x.tobytes() for x in got] == [w[0] for w in _pmap(lambda a, b: op.decaps(bits, a.tobytes(), b.tobytes()),
                                                              sk, enc)]
    assert np.array_equal(got, ss)


def test_raw_ecdh_against_openssl(bits):
    from cryptography.hazmat.primitives import serialization as ser
    from cryptography.hazmat.primitives.asymmetric import ec
    c, m = CURVES[bits], _mod(bits)
    pub = lambda k: k.public_key().public_bytes(ser.Encoding.X962, ser.PublicFormat.UncompressedPoint)  # noqa: E731
    n = 1 << 9
    ks = [ec.generate_private_key(c.ossl()) for _ in range(n)]
    ps = [ec.generate_private_key(c.ossl()) for _ in range(n)]
    sk = _rows([k.private_numbers().private_value.to_bytes(c.nbytes, "big") for k in ks])
    assert [r.tobytes() for r in getattr(m, f"p{bits}_keygen")(sk)] == [pub(k) for k in ks]
    sh = getattr(m, f"p{bits}_shared")(sk, _rows([pub(p) for p in ps]))
    assert [r.tobytes() for r in sh] == [k.exchange(ec.ECDH(), p.public_key()) for k, p in zip(ks, ps)]
    # the edges of the scalar range, from the fixed and the variable base
    N = c.n
    edge = [1, 2, 3, N - 1, N - 2, 2**(N.bit_length() - 1), 2**(N.bit_length() - 1) - 1]
    got = getattr(m, f"p{bits}_keygen")(_rows([k.to_bytes(c.nbytes, "big") for k in edge]))
    assert [r.tobytes() for r in got] == [pub(ec.derive_private_key(k, c.ossl())) for k in edge]
    peer = ec.generate_private_key(c.ossl())
    got = getattr(m, f"p{bits}_shared")(_rows([k.to_bytes(c.nbytes, "big") for k in edge]),
                                        _rows([pub(peer)] * len(edge)))
    assert [r.tobytes() for r in got] == [ec.derive_private_key(k, c.ossl()).exchange(ec.ECDH(), peer.public_key())
                                          for k in edge]


def _bad_point(bits):
    g = model.enc(CURVES[bits], CURVES[bits].g)
    return g[:-1] + bytes([g[-1] ^ 1])  # off the curve


@pytest.mark.parametrize("dev", [False, True], ids=["numpy", "cuda"])
def test_invalid_keys_inside_valid_batches(bits, dev):
    import torch
    from oracle import nistp as op
    c, m, s = CURVES[bits], _mod(bits), _scheme(bits)
    n, bad = 64, 17
    pkR, skR = _keys(bits, n, 11)
    pkS, skS = _keys(bits, n, 12)
    es = _rand(n, c.nbytes, 13)
    badp = np.frombuffer(_bad_point(bits), np.uint8)
    bads = np.frombuffer(c.n.to_bytes(c.nbytes, "big"), np.uint8)
    T = (lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()) if dev else (lambda a: a)  # noqa: E731
    H = (lambda a: a.cpu().numpy()) if dev else (lambda a: a)  # noqa: E731

    def bad_row(a, row):
        a = a.copy()
        a[bad] = row
        return a

    def check(exc, bit, call):
        with pytest.raises(exc) as ei:
            call()
        st = H(ei.value.status)
        assert st[bad] & bit and not np.delete(st, bad).any()

    cases = [
        ("pkR", m.ErrInvalidKEMPublicKey, 1, lambda: s.EncapsulateBatch(T(bad_row(pkR, badp)), T(es)),
         lambda i: op.encaps(bits, bad_row(pkR, badp)[i].tobytes(), es[i].tobytes())),
        ("skS", m.ErrInvalidKEMPrivateKey, 2, lambda: s.AuthEncapsulateBatch(T(pkR), T(bad_row(skS, bads)), T(es)),
         lambda i: op.encaps(bits, pkR[i].tobytes(), es[i].tobytes(), bad_row(skS, bads)[i].tobytes())),
    ]
    enc, ss = s.AuthEncapsulateBatch(pkR, skS, es)
    cases += [
        ("enc", m.ErrInvalidKEMPublicKey, 1, lambda: s.AuthDecapsulateBatch(T(skR), T(bad_row(enc, badp)), T(pkS)),
         lambda i: op.decaps(bits, skR[i].tobytes(), bad_row(enc, badp)[i].tobytes(), pkS[i].tobytes())),
        ("pkS", m.ErrInvalidKEMPublicKey, 1, lambda: s.AuthDecapsulateBatch(T(skR), T(enc), T(bad_row(pkS, badp))),
         lambda i: op.decaps(bits, skR[i].tobytes(), enc[i].tobytes(), bad_row(pkS, badp)[i].tobytes())),
        ("skR", m.ErrInvalidKEMPrivateKey, 2, lambda: s.DecapsulateBatch(T(bad_row(skR, bads)), T(enc)),
         lambda i: op.decaps(bits, bad_row(skR, bads)[i].tobytes(), enc[i].tobytes())),
    ]
    for name, exc, bit, call, oracle_op in cases:
        check(exc, bit, call)
        assert oracle_op(bad)[-1] & bit, name
    # raw ECDH: a bad scalar and a bad point in one batch
    ecdh_sk = bad_row(skR, bads)
    with pytest.raises(m.ErrInvalidKEMPrivateKey) as ei:
        getattr(m, f"p{bits}_shared")(T(ecdh_sk), T(bad_row(pkS, badp)))
    assert H(ei.value.status)[bad] == 3 and not np.delete(H(ei.value.status), bad).any()
    # the outputs next to the status, through the C ABI: zeros at the bad op, the oracle's results elsewhere
    from circl_b200 import _ffi
    L = _ffi.lib()
    fn = getattr(L, f"cb200_hpke_p{bits}_auth_encaps")
    st = np.zeros(n, np.uint8)
    out_ss = np.empty((n, c.nss), np.uint8)
    out_enc = np.empty((n, c.npk), np.uint8)
    p = lambda a: a.ctypes.data  # noqa: E731
    pkR_bad = bad_row(pkR, badp)
    rc = fn(p(pkR_bad), c.npk, p(skS), c.nbytes, p(es), p(out_enc), p(out_ss), p(st), n)
    assert rc == -3 and st[bad] == 1 and not out_ss[bad].any() and out_enc[bad].any()
    for i in (0, bad - 1, bad + 1, n - 1):
        assert op.encaps(bits, pkR[i].tobytes(), es[i].tobytes(), skS[i].tobytes()) == (out_enc[i].tobytes(),
                                                                                        out_ss[i].tobytes(), 0)
    skS_bad = bad_row(skS, bads)
    skS_bad[3] = 0
    rc = fn(p(pkR_bad), c.npk, p(skS_bad), c.nbytes, p(es), p(out_enc), p(out_ss), p(st), n)
    assert rc == -5 and st[bad] == 3 and st[3] == 2 and not out_ss[[3, bad]].any()


def test_invalid_shared_keys_reach_every_op(bits):
    """A shared key (stride 0) that fails marks every op, the once-computed static DH included."""
    import torch
    from circl_b200 import _ffi
    c, m, s = CURVES[bits], _mod(bits), _scheme(bits)
    n = 300
    pkR, skR = _keys(bits, n, 21)
    es = _rand(n, c.nbytes, 22)
    L = _ffi.lib()
    p = lambda a: a.ctypes.data  # noqa: E731
    bads = np.frombuffer(c.n.to_bytes(c.nbytes, "big"), np.uint8).copy()
    enc, ss, st = np.empty((n, c.npk), np.uint8), np.empty((n, c.nss), np.uint8), np.zeros(n, np.uint8)
    rc = getattr(L, f"cb200_hpke_p{bits}_auth_encaps")(p(pkR[:1].copy()), 0, p(bads), 0, p(es), p(enc), p(ss), p(st), n)
    assert rc == -5 and (st == 2).all() and not ss.any()
    badp = np.frombuffer(_bad_point(bits), np.uint8).copy()
    st[:] = 0
    rc = getattr(L, f"cb200_hpke_p{bits}_auth_encaps")(p(badp), 0, p(skR[:1].copy()), 0, p(es), p(enc), p(ss), p(st), n)
    assert rc == -3 and (st == 1).all() and not ss.any()
    st[:] = 0
    rc = getattr(L, f"cb200_hpke_p{bits}_decaps")(p(bads), 0, p(enc), p(ss), p(st), n)
    assert rc == -5 and (st & 2).all() and not ss.any()
    with pytest.raises(m.ErrInvalidKEMPrivateKey) as ei:
        s.AuthEncapsulateBatch(torch.from_numpy(pkR).cuda(), torch.from_numpy(bads[None].repeat(n, 0)).cuda(),
                               torch.from_numpy(es).cuda())
    assert (ei.value.status.cpu().numpy() == 2).all()


def test_unmarshal_validates(bits):
    c, m, s = CURVES[bits], _mod(bits), _scheme(bits)
    with pytest.raises(m.ErrInvalidKEMPublicKey):
        s.UnmarshalBinaryPublicKey(_bad_point(bits))
    with pytest.raises(m.ErrInvalidKEMPrivateKey):
        s.UnmarshalBinaryPrivateKey(c.n.to_bytes(c.nbytes, "big"))
    with pytest.raises(m.ErrInvalidKEMPublicKey):
        s.Decapsulate(s.UnmarshalBinaryPrivateKey((5).to_bytes(c.nbytes, "big")), _bad_point(bits))
    pk, sk = s.GenerateKeyPair()
    enc, ss = s.Encapsulate(pk)
    assert s.Decapsulate(sk, enc) == ss


def test_openssl_hpke_interoperability(bits):
    from cryptography.hazmat.primitives import hpke as ossl
    from cryptography.hazmat.primitives import serialization as ser
    from cryptography.hazmat.primitives.asymmetric import ec
    c, s = CURVES[bits], _scheme(bits)
    suite = ossl.Suite(ossl.KEM.P384 if bits == 384 else ossl.KEM.P521,
                       ossl.KDF.HKDF_SHA384 if bits == 384 else ossl.KDF.HKDF_SHA512, ossl.AEAD.AES_256_GCM)
    info = b"circl_b200 interop"
    keys = [ec.generate_private_key(c.ossl()) for _ in range(8)]
    cts = [suite.encrypt(b"to the gpu %d" % i, k.public_key(), info=info) for i, k in enumerate(keys)]
    sks = _rows([k.private_numbers().private_value.to_bytes(c.nbytes, "big") for k in keys])
    ss = s.DecapsulateBatch(sks, _rows([x[:c.npk] for x in cts]))
    for i, x in enumerate(cts):
        aead, nonce = model.schedule(c, ss[i].tobytes(), info)
        assert aead.decrypt(nonce, x[c.npk:], b"") == b"to the gpu %d" % i
    pks = _rows([k.public_key().public_bytes(ser.Encoding.X962, ser.PublicFormat.UncompressedPoint) for k in keys])
    enc, ss = s.EncapsulateBatch(pks, _rand(8, c.nbytes, 31))
    for i, k in enumerate(keys):
        aead, nonce = model.schedule(c, ss[i].tobytes(), info)
        sealed = enc[i].tobytes() + aead.encrypt(nonce, b"from the gpu %d" % i, b"")
        assert suite.decrypt(sealed, k, info=info) == b"from the gpu %d" % i


def test_device_pointers_at_odd_bytes(bits):
    """CUDA tensors viewed at an odd offset: rows at any byte give the host results."""
    import torch
    c, s = CURVES[bits], _scheme(bits)
    n = 257
    pk, sk = _keys(bits, n, 51)
    es = _rand(n, c.nbytes, 52)
    enc, ss = s.AuthEncapsulateBatch(pk, sk, es)
    buf = torch.zeros(n * c.npk + 1, dtype=torch.uint8, device="cuda")
    dpk = buf[1:].view(n, c.npk)
    dpk.copy_(torch.from_numpy(pk).cuda())
    kbuf = torch.zeros(n * c.nbytes + 3, dtype=torch.uint8, device="cuda")
    dsk = kbuf[3:].view(n, c.nbytes)
    dsk.copy_(torch.from_numpy(sk).cuda())
    denc, dss = s.AuthEncapsulateBatch(dpk, dsk, torch.from_numpy(es).cuda())
    assert np.array_equal(denc.cpu().numpy(), enc) and np.array_equal(dss.cpu().numpy(), ss)
    assert np.array_equal(s.AuthDecapsulateBatch(dsk, denc, dpk).cpu().numpy(), ss)


@pytest.mark.parametrize("b", [384, 521])
def test_host_batch_split_across_gpus(b):
    import circl_b200
    from circl_b200 import _ffi
    if _ffi.lib().cb200_device_count() < 2:
        pytest.skip("needs two GPUs")
    circl_b200.init_devices(0)
    try:
        from oracle import nistp as op
        s = _scheme(b)
        n = (1 << 14) + 11
        pk, sk = _keys(b, n, 41)
        es = _rand(n, CURVES[b].nbytes, 42)
        enc, ss = s.AuthEncapsulateBatch(pk, sk, es)
        assert np.array_equal(s.AuthDecapsulateBatch(sk, enc, pk), ss)
        for i in (0, n // 2 - 1, n // 2, n - 1):
            assert op.encaps(b, pk[i].tobytes(), es[i].tobytes(), sk[i].tobytes()) == (enc[i].tobytes(),
                                                                                       ss[i].tobytes(), 0)
    finally:
        circl_b200.shutdown()
