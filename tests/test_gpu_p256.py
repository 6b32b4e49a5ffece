"""GPU parity for P-256 and HPKE's DHKEM(P-256, HKDF-SHA256): the RFC 9180 vectors through the C ABI, the oracle on
2^12 random operations with per-op and shared keys in every position, raw ECDH against OpenSSL (cryptography), a seed
whose key comes from a later candidate, invalid keys inside valid batches (host arrays and CUDA tensors), OpenSSL's
HPKE in both directions, and host batches over two GPUs."""
import concurrent.futures as cf
import hashlib
import hmac

import numpy as np
import pytest

from conftest import load_golden

pytestmark = pytest.mark.gpu

NAME = "HPKE_KEM_P256_HKDF_SHA256"
N_ORDER = 0xffffffff00000000ffffffffffffffffbce6faada7179e84f3b9cac2fc632551


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


def _pmap(fn, *cols):
    """fn over rows, in threads (the oracle's ctypes calls release the GIL)."""
    with cf.ThreadPoolExecutor(16) as ex:
        return list(ex.map(fn, *cols))


def _scheme():
    from circl_b200 import p256
    return p256.ByName(NAME)


def test_rfc9180_vectors_through_the_c_abi(cb):
    s = _scheme()
    mine = load_golden("hpke_p256_vectors.json.gz")["vectors"]
    assert len(mine) == 32 and all(v["kem_id"] == 0x10 for v in mine)
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
    # the single-operation methods
    v = auth[0]
    h = lambda k: bytes.fromhex(v[k])  # noqa: E731
    pkR, skR = s.DeriveKeyPair(h("ikmR"))
    assert (pkR.MarshalBinary(), skR.MarshalBinary()) == (h("pkRm"), h("skRm"))
    assert skR.Public().MarshalBinary() == h("pkRm")
    pkS, skS = s.UnmarshalBinaryPublicKey(h("pkSm")), s.UnmarshalBinaryPrivateKey(h("skSm"))
    assert s.AuthEncapsulateDeterministically(pkR, skS, h("ikmE")) == (h("enc"), h("shared_secret"))
    assert s.AuthDecapsulate(skR, h("enc"), pkS) == h("shared_secret")
    v = base[0]
    pkR, skR = s.UnmarshalBinaryPublicKey(h("pkRm")), s.UnmarshalBinaryPrivateKey(h("skRm"))
    assert s.EncapsulateDeterministically(pkR, h("ikmE")) == (h("enc"), h("shared_secret"))
    assert s.Decapsulate(skR, h("enc")) == h("shared_secret")
    pk, sk = s.GenerateKeyPair()
    enc, ss = s.Encapsulate(pk)
    assert s.Decapsulate(sk, enc) == ss


def test_candidate_loop_seed(cb):
    """A seed whose ctr = 0 candidate is >= n: the key is the ctr = 1 candidate, on the device as in the oracle."""
    from oracle import p256 as op
    s = _scheme()
    fx = load_golden("hpke_p256_vectors.json.gz")["ctr_seeds"]
    assert fx and all(f["ctr"] > 0 for f in fx)
    seeds = _rows([bytes.fromhex(f["ikm"]) for f in fx] * 3)
    pk, sk = s.DeriveKeyPairBatch(seeds)
    for i, f in enumerate(fx * 3):
        assert (pk[i].tobytes().hex(), sk[i].tobytes().hex()) == (f["pk"], f["sk"])
        assert op.keygen(bytes.fromhex(f["ikm"])) == (bytes.fromhex(f["pk"]), bytes.fromhex(f["sk"]), f["ctr"])
    # as the ephemeral key of an encapsulation too
    enc, ss = s.EncapsulateBatch(pk[:1].repeat(len(seeds), 0), seeds)
    assert np.array_equal(enc, pk)
    assert op.encaps(pk[0].tobytes(), seeds[0].tobytes())[:2] == (enc[0].tobytes(), ss[0].tobytes())


def _keys(n, seed):
    s = _scheme()
    return s.DeriveKeyPairBatch(_rand(n, 32, seed))


@pytest.mark.parametrize("shared", ["none", "R", "S", "RS"])
def test_oracle_parity_auth(cb, shared):
    """2^12 AuthEncap / AuthDecap with pkR / skR and skS / pkS per op or shared by the batch."""
    from oracle import p256 as op
    s = _scheme()
    n = 1 << 12
    pkR, skR = _keys(n, 1)
    pkS, skS = _keys(n, 2)
    es = _rand(n, 32, 3)
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
    want = _pmap(lambda a, b, c: op.encaps(a.tobytes(), b.tobytes(), c.tobytes()), pkR, es, skS)
    assert [(e.tobytes(), x.tobytes(), 0) for e, x in zip(enc, ss)] == want
    assert np.array_equal(s.AuthDecapsulateBatch(skR_arg, enc, pkS_arg), ss)


@pytest.mark.parametrize("shared", [False, True])
def test_oracle_parity_base(cb, shared):
    from oracle import p256 as op
    s = _scheme()
    n = 1 << 12
    seeds = _rand(n, 32, 4)
    pk, sk = s.DeriveKeyPairBatch(seeds)
    got = _pmap(lambda a: op.keygen(a.tobytes())[:2], seeds)
    assert [(a.tobytes(), b.tobytes()) for a, b in zip(pk, sk)] == got
    es = _rand(n, 32, 5)
    if shared:
        pk_arg, sk_arg = s.UnmarshalBinaryPublicKey(pk[0].tobytes()), s.UnmarshalBinaryPrivateKey(sk[0].tobytes())
        pk, sk = pk[:1].repeat(n, 0), sk[:1].repeat(n, 0)
    else:
        pk_arg, sk_arg = pk, sk
    enc, ss = s.EncapsulateBatch(pk_arg, es)
    want = _pmap(lambda a, b: op.encaps(a.tobytes(), b.tobytes()), pk, es)
    assert [(e.tobytes(), x.tobytes(), 0) for e, x in zip(enc, ss)] == want
    got = s.DecapsulateBatch(sk_arg, enc)
    assert [x.tobytes() for x in got] == [w[0] for w in _pmap(lambda a, b: op.decaps(a.tobytes(), b.tobytes()), sk, enc)]
    assert np.array_equal(got, ss)


def test_raw_ecdh_against_openssl(cb):
    from cryptography.hazmat.primitives import serialization as ser
    from cryptography.hazmat.primitives.asymmetric import ec
    from circl_b200 import p256
    n = 1 << 10
    rng = np.random.default_rng(9)
    ks = [ec.derive_private_key(int(rng.integers(1, 2**62)) * 2**190 + i + 1, ec.SECP256R1()) for i in range(n)]
    ps = [ec.generate_private_key(ec.SECP256R1()) for _ in range(n)]
    sk = _rows([k.private_numbers().private_value.to_bytes(32, "big") for k in ks])
    pts = _rows([p.public_key().public_bytes(ser.Encoding.X962, ser.PublicFormat.UncompressedPoint) for p in ps])
    pub = p256.p256_keygen(sk)
    assert [r.tobytes() for r in pub] == [k.public_key().public_bytes(ser.Encoding.X962, ser.PublicFormat.UncompressedPoint)
                                          for k in ks]
    sh = p256.p256_shared(sk, pts)
    assert [r.tobytes() for r in sh] == [k.exchange(ec.ECDH(), p.public_key()) for k, p in zip(ks, ps)]
    # the edges of the scalar range, from the fixed and the variable base
    edge = _rows([k.to_bytes(32, "big") for k in (1, 2, 3, N_ORDER - 1, N_ORDER - 2, 2**255, 2**255 - 1)])
    for r, k in zip(p256.p256_keygen(edge), (1, 2, 3, N_ORDER - 1, N_ORDER - 2, 2**255, 2**255 - 1)):
        want = ec.derive_private_key(k, ec.SECP256R1()).public_key()
        assert r.tobytes() == want.public_bytes(ser.Encoding.X962, ser.PublicFormat.UncompressedPoint)


def _bad_point():
    from circl_b200 import p256
    g = p256.p256_keygen(_rows([(1).to_bytes(32, "big")]))[0].tobytes()
    return g[:64] + bytes([g[64] ^ 1])  # off the curve


@pytest.mark.parametrize("dev", [False, True], ids=["numpy", "cuda"])
def test_invalid_keys_inside_valid_batches(cb, dev):
    import torch
    from circl_b200 import p256
    from oracle import p256 as op
    s = _scheme()
    n, bad = 64, 17
    pkR, skR = _keys(n, 11)
    pkS, skS = _keys(n, 12)
    es = _rand(n, 32, 13)
    badp, bads = np.frombuffer(_bad_point(), np.uint8), np.frombuffer(N_ORDER.to_bytes(32, "big"), np.uint8)
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

    # pkR (Encap and AuthEncap): bit 0; skS: bit 1.  The ss of every other op is the oracle's.
    cases = [
        ("pkR", p256.ErrInvalidKEMPublicKey, 1,
         lambda: s.EncapsulateBatch(T(bad_row(pkR, badp)), T(es)),
         lambda i: op.encaps(bad_row(pkR, badp)[i].tobytes(), es[i].tobytes())),
        ("skS", p256.ErrInvalidKEMPrivateKey, 2,
         lambda: s.AuthEncapsulateBatch(T(pkR), T(bad_row(skS, bads)), T(es)),
         lambda i: op.encaps(pkR[i].tobytes(), es[i].tobytes(), bad_row(skS, bads)[i].tobytes())),
    ]
    enc, ss = s.AuthEncapsulateBatch(pkR, skS, es)
    cases += [
        ("enc", p256.ErrInvalidKEMPublicKey, 1,
         lambda: s.AuthDecapsulateBatch(T(skR), T(bad_row(enc, badp)), T(pkS)),
         lambda i: op.decaps(skR[i].tobytes(), bad_row(enc, badp)[i].tobytes(), pkS[i].tobytes())),
        ("pkS", p256.ErrInvalidKEMPublicKey, 1,
         lambda: s.AuthDecapsulateBatch(T(skR), T(enc), T(bad_row(pkS, badp))),
         lambda i: op.decaps(skR[i].tobytes(), enc[i].tobytes(), bad_row(pkS, badp)[i].tobytes())),
        ("skR", p256.ErrInvalidKEMPrivateKey, 2,
         lambda: s.DecapsulateBatch(T(bad_row(skR, bads)), T(enc)),
         lambda i: op.decaps(bad_row(skR, bads)[i].tobytes(), enc[i].tobytes())),
    ]
    for name, exc, bit, call, oracle_op in cases:
        check(exc, bit, call)
        assert oracle_op(bad)[-1] & bit, name  # the oracle reports the same bit
    # the outputs next to the status, through the C ABI: zeros at the bad op, the oracle's results elsewhere
    from circl_b200 import _ffi
    L = _ffi.lib()
    st = np.zeros(n, np.uint8)
    out_ss = np.empty((n, 32), np.uint8)
    out_enc = np.empty((n, 65), np.uint8)
    p = lambda a: a.ctypes.data  # noqa: E731
    pkR_bad = bad_row(pkR, badp)
    rc = L.cb200_hpke_p256_auth_encaps(p(pkR_bad), 65, p(skS), 32, p(es), p(out_enc), p(out_ss), p(st), n)
    assert rc == -3 and st[bad] == 1 and not out_ss[bad].any() and out_enc[bad].any()
    for i in (0, bad - 1, bad + 1, n - 1):
        assert op.encaps(pkR[i].tobytes(), es[i].tobytes(), skS[i].tobytes()) == (out_enc[i].tobytes(),
                                                                                   out_ss[i].tobytes(), 0)
    # both kinds in one batch: the private-key error wins
    skS_bad = bad_row(skS, bads)
    skS_bad[3] = 0
    rc = L.cb200_hpke_p256_auth_encaps(p(pkR_bad), 65, p(skS_bad), 32, p(es), p(out_enc), p(out_ss), p(st), n)
    assert rc == -5 and st[bad] == 3 and st[3] == 2 and not out_ss[[3, bad]].any()


def test_invalid_shared_keys_reach_every_op(cb):
    """A shared key (stride 0) that fails marks every op, the once-computed static DH included."""
    from circl_b200 import p256
    s = _scheme()
    n = 300
    pkR, skR = _keys(n, 21)
    es = _rand(n, 32, 22)
    zero = np.zeros(n, np.uint8)
    from circl_b200 import _ffi
    L = _ffi.lib()
    p = lambda a: a.ctypes.data  # noqa: E731
    bads = np.frombuffer(N_ORDER.to_bytes(32, "big"), np.uint8).copy()
    enc, ss, st = np.empty((n, 65), np.uint8), np.empty((n, 32), np.uint8), zero.copy()
    # skS and pkR both shared: Shared(skS, pkR) is computed once
    rc = L.cb200_hpke_p256_auth_encaps(p(pkR[:1].copy()), 0, p(bads), 0, p(es), p(enc), p(ss), p(st), n)
    assert rc == -5 and (st == 2).all() and not ss.any()
    with pytest.raises(p256.ErrInvalidKEMPrivateKey):
        s.AuthEncapsulateBatch(pkR[:1].repeat(n, 0), bads[None].repeat(n, 0), es)
    badp = np.frombuffer(_bad_point(), np.uint8).copy()
    st = zero.copy()
    rc = L.cb200_hpke_p256_auth_encaps(p(badp), 0, p(skR[:1].copy()), 0, p(es), p(enc), p(ss), p(st), n)
    assert rc == -3 and (st == 1).all() and not ss.any()
    st = zero.copy()
    rc = L.cb200_hpke_p256_decaps(p(bads), 0, p(enc), p(ss), p(st), n)
    assert rc == -5 and (st & 2).all() and not ss.any()
    import torch
    with pytest.raises(p256.ErrInvalidKEMPrivateKey) as ei:
        s.AuthEncapsulateBatch(torch.from_numpy(pkR).cuda(), torch.from_numpy(bads[None].repeat(n, 0)).cuda(),
                               torch.from_numpy(es).cuda())
    assert (ei.value.status.cpu().numpy() == 2).all()


def test_unmarshal_validates(cb):
    from circl_b200 import p256
    s = _scheme()
    with pytest.raises(p256.ErrInvalidKEMPublicKey):
        s.UnmarshalBinaryPublicKey(_bad_point())
    with pytest.raises(p256.ErrInvalidKEMPrivateKey):
        s.UnmarshalBinaryPrivateKey(N_ORDER.to_bytes(32, "big"))
    with pytest.raises(p256.ErrInvalidKEMPublicKey):
        s.Decapsulate(s.UnmarshalBinaryPrivateKey((5).to_bytes(32, "big")), _bad_point())


def _schedule(ss: bytes, info: bytes):
    """RFC 9180 section 5.1, base mode, for DHKEM(P-256) / HKDF-SHA256 / AES-128-GCM: (AESGCM(key), base_nonce)."""
    from cryptography.hazmat.primitives.ciphers.aead import AESGCM
    sid = b"HPKE" + (0x10).to_bytes(2, "big") + (1).to_bytes(2, "big") + (1).to_bytes(2, "big")
    ext = lambda salt, lab, ikm: hmac.new(salt or bytes(32), b"HPKE-v1" + sid + lab + ikm, hashlib.sha256).digest()  # noqa: E731
    exp = lambda prk, lab, inf, L: hmac.new(prk, L.to_bytes(2, "big") + b"HPKE-v1" + sid + lab + inf + b"\x01",  # noqa: E731
                                            hashlib.sha256).digest()[:L]
    ctx = b"\x00" + ext(b"", b"psk_id_hash", b"") + ext(b"", b"info_hash", info)
    secret = ext(ss, b"secret", b"")
    return AESGCM(exp(secret, b"key", ctx, 16)), exp(secret, b"base_nonce", ctx, 12)


def test_openssl_hpke_interoperability(cb):
    from cryptography.hazmat.primitives import hpke as ossl
    from cryptography.hazmat.primitives import serialization as ser
    from cryptography.hazmat.primitives.asymmetric import ec
    s = _scheme()
    suite = ossl.Suite(ossl.KEM.P256, ossl.KDF.HKDF_SHA256, ossl.AEAD.AES_128_GCM)
    info = b"circl_b200 interop"
    keys = [ec.generate_private_key(ec.SECP256R1()) for _ in range(8)]
    cts = [suite.encrypt(b"to the gpu %d" % i, k.public_key(), info=info) for i, k in enumerate(keys)]
    sks = _rows([k.private_numbers().private_value.to_bytes(32, "big") for k in keys])
    ss = s.DecapsulateBatch(sks, _rows([c[:65] for c in cts]))
    for i, c in enumerate(cts):
        aead, nonce = _schedule(ss[i].tobytes(), info)
        assert aead.decrypt(nonce, c[65:], b"") == b"to the gpu %d" % i
    pks = _rows([k.public_key().public_bytes(ser.Encoding.X962, ser.PublicFormat.UncompressedPoint) for k in keys])
    enc, ss = s.EncapsulateBatch(pks, _rand(8, 32, 31))
    for i, k in enumerate(keys):
        aead, nonce = _schedule(ss[i].tobytes(), info)
        sealed = enc[i].tobytes() + aead.encrypt(nonce, b"from the gpu %d" % i, b"")
        assert suite.decrypt(sealed, k, info=info) == b"from the gpu %d" % i


def test_device_pointers_at_odd_bytes(cb):
    """CUDA tensors viewed at an odd offset: rows of 65 bytes at any byte give the host results."""
    import torch
    s = _scheme()
    n = 257
    pk, sk = _keys(n, 51)
    es = _rand(n, 32, 52)
    enc, ss = s.AuthEncapsulateBatch(pk, sk, es)
    buf = torch.zeros(n * 65 + 1, dtype=torch.uint8, device="cuda")
    dpk = buf[1:].view(n, 65)
    dpk.copy_(torch.from_numpy(pk).cuda())
    denc, dss = s.AuthEncapsulateBatch(dpk, torch.from_numpy(sk).cuda(), torch.from_numpy(es).cuda())
    assert np.array_equal(denc.cpu().numpy(), enc) and np.array_equal(dss.cpu().numpy(), ss)


def test_host_batch_split_across_gpus():
    import circl_b200
    from circl_b200 import _ffi
    if _ffi.lib().cb200_device_count() < 2:
        pytest.skip("needs two GPUs")
    circl_b200.init_devices(0)
    try:
        from oracle import p256 as op
        s = _scheme()
        n = (1 << 15) + 11
        pk, sk = s.DeriveKeyPairBatch(_rand(n, 32, 41))
        es = _rand(n, 32, 42)
        enc, ss = s.AuthEncapsulateBatch(pk, sk, es)
        assert np.array_equal(s.AuthDecapsulateBatch(sk, enc, pk), ss)
        for i in (0, n // 2 - 1, n // 2, n - 1):
            assert op.encaps(pk[i].tobytes(), es[i].tobytes(), sk[i].tobytes()) == (enc[i].tobytes(), ss[i].tobytes(), 0)
    finally:
        circl_b200.shutdown()

