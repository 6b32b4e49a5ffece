"""GPU parity for HPKE's DHKEM(X25519, HKDF-SHA256) and DHKEM(X448, HKDF-SHA512): the RFC 9180 vectors through the C
ABI, the oracle on 2^12 random operations with per-op and shared keys, low-order shares in every key position, bit 255
of X25519 keys in kem_context, device pointers, OpenSSL's HPKE in both directions, and host batches over two GPUs."""
import hashlib
import hmac

import numpy as np
import pytest

import hpke_model as M
from conftest import load_golden

pytestmark = pytest.mark.gpu

IDS = [M.X25519_ID, M.X448_ID]
NAME = {M.X25519_ID: "HPKE_KEM_X25519_HKDF_SHA256", M.X448_ID: "HPKE_KEM_X448_HKDF_SHA512"}


@pytest.fixture(scope="module")
def cb():
    import circl_b200
    circl_b200.init(0)
    yield circl_b200
    circl_b200.shutdown()


def _rows(bs):
    return np.stack([np.frombuffer(bytes(b), dtype=np.uint8) for b in bs])


def _rand(n, w, seed):
    return np.random.default_rng(seed).integers(0, 256, size=(n, w), dtype=np.uint8)


def test_rfc9180_vectors_through_the_c_abi(cb):
    from circl_b200 import hpke
    vs = load_golden("hpke_vectors.json.gz")["vectors"]
    for kid in IDS:
        s = hpke.ByName(NAME[kid])
        mine = [v for v in vs if v["kem_id"] == kid]
        b = lambda k: _rows([bytes.fromhex(v[k]) for v in mine])  # noqa: E731
        for who in "ER":
            pk, sk = s.DeriveKeyPairBatch(b("ikm" + who))
            assert np.array_equal(pk, b(f"pk{who}m")) and np.array_equal(sk, b(f"sk{who}m"))
        auth = [v for v in mine if v["mode"] in (2, 3)]
        ba = lambda k: _rows([bytes.fromhex(v[k]) for v in auth])  # noqa: E731
        pk, sk = s.DeriveKeyPairBatch(ba("ikmS"))
        assert np.array_equal(pk, ba("pkSm")) and np.array_equal(sk, ba("skSm"))
        # base / psk modes use Encap / Decap, auth / auth-psk AuthEncap / AuthDecap
        base = [v for v in mine if v["mode"] in (0, 1)]
        bb = lambda k: _rows([bytes.fromhex(v[k]) for v in base])  # noqa: E731
        enc, ss = s.EncapsulateBatch(bb("pkRm"), bb("ikmE"))
        assert np.array_equal(enc, bb("enc")) and np.array_equal(ss, bb("shared_secret"))
        assert np.array_equal(s.DecapsulateBatch(bb("skRm"), bb("enc")), bb("shared_secret"))
        enc, ss = s.AuthEncapsulateBatch(ba("pkRm"), ba("skSm"), ba("ikmE"))
        assert np.array_equal(enc, ba("enc")) and np.array_equal(ss, ba("shared_secret"))
        assert np.array_equal(s.AuthDecapsulateBatch(ba("skRm"), ba("enc"), ba("pkSm")), ba("shared_secret"))
        # the single-operation methods
        v = auth[0]
        h = lambda k: bytes.fromhex(v[k])  # noqa: E731
        pkR, skR = s.DeriveKeyPair(h("ikmR"))
        pkS, skS = s.DeriveKeyPair(h("ikmS"))
        assert skR.Public().Equal(pkR) and pkR.MarshalBinary() == h("pkRm")
        enc, ss = s.AuthEncapsulateDeterministically(pkR, skS, h("ikmE"))
        assert (enc, ss) == (h("enc"), h("shared_secret"))
        assert s.AuthDecapsulate(skR, enc, pkS) == ss


@pytest.mark.parametrize("kid", IDS)
def test_oracle_parity_per_op_and_shared_keys(cb, kid):
    from oracle import hpke as oh
    from circl_b200 import hpke
    s, n, N = hpke.ByName(NAME[kid]), 1 << 12, M.KEMS[kid].n
    seedsR, seedsS, eseeds = _rand(n, N, kid), _rand(n, N, kid + 1), _rand(n, N, kid + 2)
    pkR, skR = s.DeriveKeyPairBatch(seedsR)
    pkS, skS = s.DeriveKeyPairBatch(seedsS)
    for i in range(n):
        assert (pkR[i].tobytes(), skR[i].tobytes()) == oh.keygen(kid, seedsR[i].tobytes())
    enc, ss = s.EncapsulateBatch(pkR, eseeds)
    dss = s.DecapsulateBatch(skR, enc)
    aenc, ass = s.AuthEncapsulateBatch(pkR, skS, eseeds)
    adss = s.AuthDecapsulateBatch(skR, aenc, pkS)
    assert np.array_equal(enc, aenc) and np.array_equal(ss, dss) and np.array_equal(ass, adss)
    for i in range(n):
        r, e, sS = pkR[i].tobytes(), eseeds[i].tobytes(), skS[i].tobytes()
        assert oh.encaps(kid, r, e) == (enc[i].tobytes(), ss[i].tobytes(), 0)
        assert oh.encaps(kid, r, e, sS) == (aenc[i].tobytes(), ass[i].tobytes(), 0)
    # one key for the whole batch, in each key position (stride 0); checked against the oracle on every 8th op
    k0R = s.UnmarshalBinaryPublicKey(pkR[0].tobytes())
    s0R = s.UnmarshalBinaryPrivateKey(skR[0].tobytes())
    k0S = s.UnmarshalBinaryPublicKey(pkS[0].tobytes())
    s0S = s.UnmarshalBinaryPrivateKey(skS[0].tobytes())
    e1, ss1 = s.EncapsulateBatch(k0R, eseeds)
    e2, ss2 = s.AuthEncapsulateBatch(k0R, skS, eseeds)
    e3, ss3 = s.AuthEncapsulateBatch(pkR, s0S, eseeds)
    d1 = s.DecapsulateBatch(s0R, e1)
    d2 = s.AuthDecapsulateBatch(s0R, e2, pkS)
    d3 = s.AuthDecapsulateBatch(skR, e3, k0S)
    assert np.array_equal(d1, ss1) and np.array_equal(d2, ss2) and np.array_equal(d3, ss3)
    assert np.array_equal(s.DecapsulateBatch(s0R, enc[:64])[:64], s.DecapsulateBatch(np.repeat(skR[:1], 64, 0), enc[:64]))
    for i in range(0, n, 8):
        e = eseeds[i].tobytes()
        assert oh.encaps(kid, pkR[0].tobytes(), e) == (e1[i].tobytes(), ss1[i].tobytes(), 0)
        assert oh.encaps(kid, pkR[0].tobytes(), e, skS[i].tobytes()) == (e2[i].tobytes(), ss2[i].tobytes(), 0)
        assert oh.encaps(kid, pkR[i].tobytes(), e, skS[0].tobytes()) == (e3[i].tobytes(), ss3[i].tobytes(), 0)
        assert oh.decaps(kid, skR[i].tobytes(), e3[i].tobytes(), pkS[0].tobytes()) == (d3[i].tobytes(), 0)


@pytest.mark.parametrize("kid", IDS)
def test_low_order_shares(cb, kid):
    from oracle import hpke as oh
    from circl_b200 import hpke
    s, N = hpke.ByName(NAME[kid]), M.KEMS[kid].n
    bad = M.low_order_points(kid)
    n = 4 * len(bad)
    pkR, skR = s.DeriveKeyPairBatch(_rand(n, N, 7))
    pkS, skS = s.DeriveKeyPairBatch(_rand(n, N, 8))
    es = _rand(n, N, 9)
    rows = np.arange(0, n, 4)  # every 4th op gets a low-order share
    want = np.zeros(n, dtype=bool)
    want[rows] = True
    for pos in ("pkR", "enc", "pkS"):
        R, S = pkR.copy(), pkS.copy()
        if pos == "pkR":
            R[rows] = _rows(bad)
        if pos == "pkS":
            S[rows] = _rows(bad)
        enc, _ = s.EncapsulateBatch(pkR, es)
        if pos == "enc":
            enc[rows] = _rows(bad)
        calls = []
        if pos == "pkR":
            calls = [lambda: s.EncapsulateBatch(R, es), lambda: s.AuthEncapsulateBatch(R, skS, es)]
        elif pos == "enc":
            calls = [lambda: s.DecapsulateBatch(skR, enc), lambda: s.AuthDecapsulateBatch(skR, enc, S)]
        else:
            calls = [lambda: s.AuthDecapsulateBatch(skR, enc, S)]
        for c in calls:
            with pytest.raises(hpke.ErrInvalidKEMSharedSecret) as ei:
                c()
            assert np.array_equal(ei.value.status != 0, want), pos
        # the results of a failed host batch: rerun through the C ABI to read ss as well
        from circl_b200._ffi import lib
        L = lib()
        ss = np.empty((n, s.SharedKeySize()), dtype=np.uint8)
        st = np.zeros(n, dtype=np.uint8)
        if pos == "pkR":
            e2 = np.empty((n, N), dtype=np.uint8)
            rc = L.cb200_hpke_auth_encaps(kid, R.ctypes.data, N, skS.ctypes.data, N, es.ctypes.data, e2.ctypes.data,
                                          ss.ctypes.data, st.ctypes.data, n)
            ref = [oh.encaps(kid, R[i].tobytes(), es[i].tobytes(), skS[i].tobytes()) for i in range(n)]
            assert all(e2[i].tobytes() == ref[i][0] for i in range(n))
            ref = [(r[1], r[2]) for r in ref]
        else:
            rc = L.cb200_hpke_auth_decaps(kid, skR.ctypes.data, N, enc.ctypes.data, S.ctypes.data, N, ss.ctypes.data,
                                          st.ctypes.data, n)
            ref = [oh.decaps(kid, skR[i].tobytes(), enc[i].tobytes(), S[i].tobytes()) for i in range(n)]
        assert rc == -3 and np.array_equal(st != 0, want)
        for i in range(n):
            assert (ss[i].tobytes(), int(st[i])) == ref[i], (pos, i)
            assert (ss[i].tobytes() == bytes(s.SharedKeySize())) == want[i]


def test_bit_255_of_x25519_keys_enters_kem_context(cb):
    from oracle import hpke as oh
    from circl_b200 import hpke
    s = hpke.ByName(NAME[M.X25519_ID])
    pkR, skR = s.DeriveKeyPairBatch(_rand(64, 32, 3))
    hi = pkR.copy()
    hi[:, 31] |= 0x80
    es = _rand(64, 32, 4)
    e1, ss1 = s.EncapsulateBatch(pkR, es)
    e2, ss2 = s.EncapsulateBatch(hi, es)
    assert np.array_equal(e1, e2) and not (ss1 == ss2).all(axis=1).any()
    for i in range(64):
        assert oh.encaps(M.X25519_ID, hi[i].tobytes(), es[i].tobytes()) == (e2[i].tobytes(), ss2[i].tobytes(), 0)
    ehi = e1.copy()
    ehi[:, 31] |= 0x80
    d = s.DecapsulateBatch(skR, ehi)
    assert not (d == ss1).all(axis=1).any()
    for i in range(64):
        assert oh.decaps(M.X25519_ID, skR[i].tobytes(), ehi[i].tobytes()) == (d[i].tobytes(), 0)


@pytest.mark.parametrize("kid", IDS)
def test_device_pointers(cb, kid):
    import torch
    from circl_b200 import hpke
    from circl_b200._ffi import lib
    s, n, N = hpke.ByName(NAME[kid]), 3000, M.KEMS[kid].n
    seeds, es = _rand(n, N, 21), _rand(n, N, 22)
    bad = M.low_order_points(kid)
    hpk, hsk = s.DeriveKeyPairBatch(seeds)
    henc, hss = s.EncapsulateBatch(hpk, es)
    dseeds, des = torch.from_numpy(seeds).cuda(), torch.from_numpy(es).cuda()
    pk, sk = s.DeriveKeyPairBatch(dseeds)
    assert pk.is_cuda and np.array_equal(pk.cpu().numpy(), hpk) and np.array_equal(sk.cpu().numpy(), hsk)
    enc, ss = s.EncapsulateBatch(pk, des)
    assert np.array_equal(enc.cpu().numpy(), henc) and np.array_equal(ss.cpu().numpy(), hss)
    assert torch.equal(s.DecapsulateBatch(sk, enc), ss)
    s0 = s.UnmarshalBinaryPrivateKey(hsk[5].tobytes())
    p0 = s.UnmarshalBinaryPublicKey(hpk[5].tobytes())
    aenc, ass = s.AuthEncapsulateBatch(p0, sk, des)
    assert torch.equal(s.AuthDecapsulateBatch(s0, aenc, pk), ass)
    assert np.array_equal(ass.cpu().numpy(), s.AuthEncapsulateBatch(p0, hsk, es)[1])
    # a device call reports failures through status only, and needs it
    enc2 = enc.clone()
    enc2[:len(bad)] = torch.from_numpy(_rows(bad)).cuda()
    st = torch.zeros(n, dtype=torch.uint8, device="cuda")
    out = torch.empty((n, s.SharedKeySize()), dtype=torch.uint8, device="cuda")
    L = lib()
    assert L.cb200_hpke_decaps(kid, sk.data_ptr(), N, enc2.data_ptr(), out.data_ptr(), st.data_ptr(), n) == 0
    torch.cuda.synchronize()
    assert st[:len(bad)].tolist() == [1] * len(bad) and st[len(bad):].sum().item() == 0
    assert out[:len(bad)].sum().item() == 0 and torch.equal(out[len(bad):], ss[len(bad):])
    assert L.cb200_hpke_decaps(kid, sk.data_ptr(), N, enc2.data_ptr(), out.data_ptr(), None, n) == -1
    assert "status" in L.cb200_last_error().decode()
    torch.cuda.synchronize()


@pytest.mark.parametrize("kid", IDS)
def test_device_tensor_failures_raise(cb, kid):
    """A device-pointer call reports low-order shares only through status; the Python methods read it back and raise
    ErrInvalidKEMSharedSecret with .status, as for host arrays, so an all-zero secret is never returned silently."""
    import torch
    from circl_b200 import hpke
    s, n, N = hpke.ByName(NAME[kid]), 256, M.KEMS[kid].n
    bad = torch.from_numpy(_rows(M.low_order_points(kid))).cuda()
    nb = bad.shape[0]
    want = torch.zeros(n, dtype=torch.bool, device="cuda")
    want[:nb] = True
    pk, sk = s.DeriveKeyPairBatch(torch.from_numpy(_rand(n, N, 51)).cuda())
    es = torch.from_numpy(_rand(n, N, 52)).cuda()
    enc, ss = s.EncapsulateBatch(pk, es)
    s0 = s.UnmarshalBinaryPrivateKey(sk[0].cpu().numpy().tobytes())
    p0 = s.UnmarshalBinaryPublicKey(pk[0].cpu().numpy().tobytes())
    encb = enc.clone()
    encb[:nb] = bad
    pkb = pk.clone()
    pkb[:nb] = bad
    calls = {"decaps enc": lambda: s.DecapsulateBatch(sk, encb),
             "decaps enc, shared skR": lambda: s.DecapsulateBatch(s0, encb),
             "auth decaps enc": lambda: s.AuthDecapsulateBatch(sk, encb, pk),
             "auth decaps pkS": lambda: s.AuthDecapsulateBatch(sk, enc, pkb),
             "auth decaps pkS, shared skR": lambda: s.AuthDecapsulateBatch(s0, enc, pkb),
             "encaps pkR": lambda: s.EncapsulateBatch(pkb, es),
             "auth encaps pkR": lambda: s.AuthEncapsulateBatch(pkb, sk, es),
             "auth encaps pkR, shared skS": lambda: s.AuthEncapsulateBatch(pkb, s0, es)}
    for what, call in calls.items():
        with pytest.raises(hpke.ErrInvalidKEMSharedSecret) as ei:
            call()
        st = ei.value.status
        assert st.is_cuda and torch.equal(st != 0, want), what
    # one low-order pkR shared by the batch fails every operation, also with a shared skS
    pb = s.UnmarshalBinaryPublicKey(bad[0].cpu().numpy().tobytes())
    for call in (lambda: s.EncapsulateBatch(pb, es), lambda: s.AuthEncapsulateBatch(pb, s0, es)):
        with pytest.raises(hpke.ErrInvalidKEMSharedSecret) as ei:
            call()
        assert bool(ei.value.status.all())
    # and a clean batch raises nothing
    assert torch.equal(s.AuthDecapsulateBatch(s0, s.AuthEncapsulateBatch(p0, s0, es)[0], p0),
                       s.AuthEncapsulateBatch(p0, s0, es)[1])


@pytest.mark.parametrize("kid", IDS)
def test_auth_encaps_with_both_keys_shared(cb, kid):
    """pkR and skS both shared: Shared(skS, pkR) is computed once for the batch; every op still matches the oracle."""
    from oracle import hpke as oh
    from circl_b200 import hpke
    s, n, N = hpke.ByName(NAME[kid]), 1000, M.KEMS[kid].n
    pk, sk = s.DeriveKeyPairBatch(_rand(2, N, 61))
    es = _rand(n, N, 62)
    pR, sS = s.UnmarshalBinaryPublicKey(pk[0].tobytes()), s.UnmarshalBinaryPrivateKey(sk[1].tobytes())
    enc, ss = s.AuthEncapsulateBatch(pR, sS, es)
    for i in range(0, n, 7):
        assert oh.encaps(kid, pk[0].tobytes(), es[i].tobytes(), sk[1].tobytes()) == (enc[i].tobytes(), ss[i].tobytes(), 0)
    assert np.array_equal(s.AuthDecapsulateBatch(s.UnmarshalBinaryPrivateKey(sk[0].tobytes()), enc,
                                                 s.UnmarshalBinaryPublicKey(pk[1].tobytes())), ss)
    # with device pointers too
    import torch
    denc, dss = s.AuthEncapsulateBatch(pR, sS, torch.from_numpy(es).cuda())
    assert np.array_equal(denc.cpu().numpy(), enc) and np.array_equal(dss.cpu().numpy(), ss)


def _schedule(ss: bytes, info: bytes):
    """RFC 9180 section 5.1, base mode, for DHKEM(X25519) / HKDF-SHA256 / AES-128-GCM: (AESGCM(key), base_nonce)."""
    from cryptography.hazmat.primitives.ciphers.aead import AESGCM
    sid = b"HPKE" + (0x20).to_bytes(2, "big") + (1).to_bytes(2, "big") + (1).to_bytes(2, "big")
    ext = lambda salt, lab, ikm: hmac.new(salt or bytes(32), b"HPKE-v1" + sid + lab + ikm, hashlib.sha256).digest()  # noqa: E731
    exp = lambda prk, lab, inf, L: hmac.new(prk, L.to_bytes(2, "big") + b"HPKE-v1" + sid + lab + inf + b"\x01",  # noqa: E731
                                            hashlib.sha256).digest()[:L]
    ctx = b"\x00" + ext(b"", b"psk_id_hash", b"") + ext(b"", b"info_hash", info)
    secret = ext(ss, b"secret", b"")
    return AESGCM(exp(secret, b"key", ctx, 16)), exp(secret, b"base_nonce", ctx, 12)


def test_openssl_hpke_interoperability(cb):
    from cryptography.hazmat.primitives import hpke as ossl
    from cryptography.hazmat.primitives.asymmetric import x25519
    from circl_b200 import hpke
    s = hpke.ByName(NAME[M.X25519_ID])
    suite = ossl.Suite(ossl.KEM.X25519, ossl.KDF.HKDF_SHA256, ossl.AEAD.AES_128_GCM)
    info = b"circl_b200 interop"
    keys = [x25519.X25519PrivateKey.generate() for _ in range(8)]
    # OpenSSL seals, the GPU decapsulates and the key schedule above opens
    cts = [suite.encrypt(b"to the gpu %d" % i, k.public_key(), info=info) for i, k in enumerate(keys)]
    sks = _rows([k.private_bytes_raw() for k in keys])
    ss = s.DecapsulateBatch(sks, _rows([c[:32] for c in cts]))
    for i, c in enumerate(cts):
        aead, nonce = _schedule(ss[i].tobytes(), info)
        assert aead.decrypt(nonce, c[32:], b"") == b"to the gpu %d" % i
    # the GPU encapsulates, the key schedule seals and OpenSSL opens
    pks = _rows([k.public_key().public_bytes_raw() for k in keys])
    enc, ss = s.EncapsulateBatch(pks, _rand(8, 32, 31))
    for i, k in enumerate(keys):
        aead, nonce = _schedule(ss[i].tobytes(), info)
        sealed = enc[i].tobytes() + aead.encrypt(nonce, b"from the gpu %d" % i, b"")
        assert suite.decrypt(sealed, k, info=info) == b"from the gpu %d" % i


def test_host_batch_split_across_gpus():
    import circl_b200
    from circl_b200 import _ffi
    if _ffi.lib().cb200_device_count() < 2:
        pytest.skip("needs two GPUs")
    circl_b200.init_devices(0)
    try:
        from oracle import hpke as oh
        from circl_b200 import hpke
        for kid in IDS:
            s, N, n = hpke.ByName(NAME[kid]), M.KEMS[kid].n, (1 << 15) + 11
            pk, sk = s.DeriveKeyPairBatch(_rand(n, N, 41))
            es = _rand(n, N, 42)
            enc, ss = s.AuthEncapsulateBatch(pk, sk, es)
            assert np.array_equal(s.AuthDecapsulateBatch(sk, enc, pk), ss)
            for i in (0, n // 2 - 1, n // 2, n - 1):
                assert oh.encaps(kid, pk[i].tobytes(), es[i].tobytes(), sk[i].tobytes()) == (enc[i].tobytes(),
                                                                                            ss[i].tobytes(), 0)
    finally:
        circl_b200.shutdown()
