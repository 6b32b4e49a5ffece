"""GPU parity for sign/ed448 and sign/eddilithium3: the reference's RFC 8032 and Wycheproof vectors, OpenSSL's Ed448 on
random batches (shared and per-op keys), contexts up to 255 bytes against the oracle and the 256-byte errors, the
private key's public half used as given, the torsion and encoding cases with the verdicts of the reference's
equation, tampered signatures, host pointers and device rows at odd byte offsets, and Ed448-Dilithium3 against the
oracle and rebuilt from OpenSSL Ed448, hashlib's SHAKE256 and the oracle's round-3 Dilithium3."""
import ctypes as C
import hashlib

import numpy as np
import pytest

import ed448_model as M
from conftest import load_golden

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cb():
    import circl_b200
    circl_b200.init(0)
    yield circl_b200
    circl_b200.shutdown()


def _rows(items):
    return np.frombuffer(b"".join(items), dtype=np.uint8).reshape(len(items), -1)


def _h(tag, i, n=57):
    return hashlib.shake_256(bytes([tag]) + i.to_bytes(8, "little")).digest(n)


def _ossl(seed):
    from cryptography.hazmat.primitives.asymmetric.ed448 import Ed448PrivateKey
    return Ed448PrivateKey.from_private_bytes(seed)


def _batch(n, tag):
    lens = [0, 1, 25, 26, 69, 70, 79, 80, 135, 136, 137, 32, 1000]
    seeds = [_h(tag, i) for i in range(n)]
    msgs = [_h(tag + 1, i, lens[i % len(lens)]) if lens[i % len(lens)] else b"" for i in range(n)]
    return seeds, msgs


def test_reference_vectors(cb):
    from circl_b200.ed448 import Ed448, SignatureOpts
    v = load_golden("ed448_vectors.json.gz")
    s = Ed448()
    for t in v["rfc8032"]:
        seed, pk, msg, sig, ctx = (bytes.fromhex(t[k]) for k in ("seed", "pk", "msg", "sig", "ctx"))
        gpk, gsk = s.DeriveKey(seed)
        assert gpk._packed == pk and gsk._packed == seed + pk
        assert s.Sign(gsk, msg, SignatureOpts(ctx)) == sig
        assert s.Verify(gpk, msg, sig, SignatureOpts(ctx))
    w = v["wycheproof"]
    assert len(w) == 86
    got = [s.Verify(s.UnmarshalBinaryPublicKey(bytes.fromhex(t["pk"])), bytes.fromhex(t["msg"]), bytes.fromhex(t["sig"]))
           for t in w]
    assert got == [t["valid"] for t in w]
    full = [i for i, t in enumerate(w) if len(t["sig"]) == 228]  # the same through one batch
    ok = s.VerifyBatch(_rows([bytes.fromhex(w[i]["pk"]) for i in full]), [bytes.fromhex(w[i]["msg"]) for i in full],
                       _rows([bytes.fromhex(w[i]["sig"]) for i in full]))
    assert list(ok) == [w[i]["valid"] for i in full]


def test_openssl_parity_per_op_and_shared_keys(cb):
    from circl_b200.ed448 import Ed448
    from oracle import ed448 as oe
    s = Ed448()
    n = 1 << 13
    seeds, msgs = _batch(n, 10)
    pk, sk = s.DeriveKeyBatch(_rows(seeds))
    sig = s.SignBatch(sk, msgs)
    for i in list(range(0, n, 97)) + [n - 1]:
        k = _ossl(seeds[i])
        assert pk[i].tobytes() == k.public_key().public_bytes_raw()
        assert sig[i].tobytes() == k.sign(msgs[i])
    for i in range(0, n, 1601):
        assert (pk[i].tobytes(), sk[i].tobytes()) == oe.ed448_keygen(seeds[i])
        assert sig[i].tobytes() == oe.ed448_sign(sk[i].tobytes(), msgs[i])
    assert s.VerifyBatch(pk, msgs, sig).all()
    key = s.UnmarshalBinaryPrivateKey(sk[7].tobytes())  # one shared key
    sig1 = s.SignBatch(key, msgs[:2048])
    for i in range(0, 2048, 211):
        assert sig1[i].tobytes() == _ossl(seeds[7]).sign(msgs[i])
    assert s.VerifyBatch(s.UnmarshalBinaryPublicKey(pk[7].tobytes()), msgs[:2048], sig1).all()


def test_contexts(cb):
    from circl_b200._ffi import lib
    from circl_b200.ed448 import Ed448, ErrContextTooLong
    from oracle import ed448 as oe
    s = Ed448()
    n = 64
    seeds, msgs = _batch(n, 20)
    pk, sk = s.DeriveKeyBatch(_rows(seeds))
    for ctx in (b"\0", b"ctx", bytes(range(255))):
        sig = s.SignBatch(sk, msgs, ctx)
        for i in range(0, n, 9):
            assert sig[i].tobytes() == oe.ed448_sign(sk[i].tobytes(), msgs[i], ctx)
        assert s.VerifyBatch(pk, msgs, sig, ctx).all()
        assert not s.VerifyBatch(pk, msgs, sig, ctx[:-1]).any()
        assert not s.VerifyBatch(pk, msgs, sig).any()
    sig = s.SignBatch(sk, msgs, bytes(255))
    # 256 bytes: the C call refuses to sign, and verification is false for every op
    ctx = np.zeros(256, dtype=np.uint8)
    blob = np.frombuffer(b"".join(msgs) + bytes(8), dtype=np.uint8)
    off = np.zeros(n + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(m) for m in msgs])
    out = np.zeros((n, 114), dtype=np.uint8)
    assert lib().cb200_ed448_sign(sk.ctypes.data, 114, blob.ctypes.data, off.ctypes.data, ctx.ctypes.data, 256,
                                  out.ctypes.data, n) == -1
    ok = np.ones(n, dtype=np.uint8)
    assert lib().cb200_ed448_verify(pk.ctypes.data, 57, blob.ctypes.data, off.ctypes.data, ctx.ctypes.data, 256,
                                    sig.ctypes.data, ok.ctypes.data, n) == 0
    assert not ok.any()
    with pytest.raises(ErrContextTooLong):
        s.SignBatch(sk, msgs, bytes(256))
    assert not s.VerifyBatch(pk, msgs, sig, bytes(256)).any()


def test_public_half_of_the_key_is_used_as_given(cb):
    from circl_b200.ed448 import Ed448
    s = Ed448()
    seed, other = _h(21, 0), _h(21, 1)
    wrong = M.public(other)
    sig = s.SignBatch(_rows([seed + wrong]), [b"message"])[0].tobytes()
    assert sig == M.sign(seed, wrong, b"message")
    assert sig != _ossl(seed).sign(b"message")
    assert not s.VerifyBatch(_rows([M.public(seed)]), [b"message"], _rows([sig]))[0]


def test_torsion_and_encoding_cases(cb):
    """Verdicts of the reference's equation (Python integers), which the oracle reproduces through the isogeny."""
    from circl_b200.ed448 import Ed448
    from oracle import ed448 as oe
    cases = M.torsion_cases()
    s = Ed448()
    ok = s.VerifyBatch(_rows([c[1] for c in cases]), [c[2] for c in cases], _rows([c[3] for c in cases]))
    assert [bool(x) for x in ok] == [c[5] for c in cases], [c[0] for c in cases]
    assert [oe.ed448_verify(c[1], c[2], c[3]) for c in cases] == [c[5] for c in cases]


def test_torsion_public_keys_sign_and_verify(cb):
    """pk = encode([s] G + T) for T of order 2 and 4: the device signs with it as given, and the signature verifies."""
    from circl_b200.ed448 import Ed448
    s = Ed448()
    seeds = [_h(22, i) for i in range(3)]
    sks, pks, msgs = [], [], []
    for j, seed in enumerate(seeds):
        sc = M.expand(seed)[0]
        pk = M.encode(M.add(M.mul(sc, M.G), M.TORSION[1 + j]))
        sks.append(seed + pk)
        pks.append(pk)
        msgs.append(b"torsion %d" % j)
    sig = s.SignBatch(_rows(sks), msgs)
    assert [sig[j].tobytes() for j in range(3)] == [M.sign(seeds[j], pks[j], msgs[j]) for j in range(3)]
    assert s.VerifyBatch(_rows(pks), msgs, sig).all()


def test_tampered_signatures(cb):
    from circl_b200.ed448 import Ed448
    s = Ed448()
    n = 300
    seeds, msgs = _batch(n, 30)
    pk, sk = s.DeriveKeyBatch(_rows(seeds))
    sig = s.SignBatch(sk, msgs).copy()
    pk2, msgs2 = pk.copy(), list(msgs)
    want = np.ones(n, dtype=bool)
    for i in range(0, n, 5):
        kind = (i // 5) % 6
        if kind == 0:
            sig[i, 3] ^= 0x10                      # R
        elif kind == 1:
            sig[i, 70] ^= 0x01                     # S
        elif kind == 2:                            # S + l: same point equation, but not canonical
            S = int.from_bytes(sig[i, 57:].tobytes(), "little") + M.L
            sig[i, 57:] = np.frombuffer(S.to_bytes(57, "little"), dtype=np.uint8)
        elif kind == 3:
            pk2[i] = np.frombuffer(M.public(_h(31, i)), dtype=np.uint8)  # another key
        elif kind == 4:
            msgs2[i] = msgs2[i] + b"\0"            # message
        else:
            pk2[i, 56] ^= 0x80                     # A with the other sign of x
        want[i] = False
    assert np.array_equal(s.VerifyBatch(pk2, msgs2, sig), want)


def test_device_pointers_at_odd_offsets(cb):
    import torch
    from circl_b200._ffi import check, lib
    from circl_b200.ed448 import Ed448
    n = 2048
    seeds, msgs = _batch(n, 40)
    blob = np.frombuffer(b"".join(msgs) + b"\0" * 8, dtype=np.uint8)
    off = np.zeros(n + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(m) for m in msgs])
    check(lib().cb200_set_stream(C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    d_blob, d_off = torch.from_numpy(blob.copy()).cuda(), torch.from_numpy(off.view(np.int64).copy()).cuda()
    # seeds, keys and signatures in rows with odd strides at odd offsets
    d_seeds = torch.zeros((n * 59 + 3,), dtype=torch.uint8, device="cuda")
    d_seeds[3:].view(n, 59)[:, :57] = torch.from_numpy(_rows(seeds).copy()).cuda()
    d_pk = torch.zeros((n * 57 + 1,), dtype=torch.uint8, device="cuda")
    d_sk = torch.zeros((n * 114 + 5,), dtype=torch.uint8, device="cuda")
    d_sig = torch.zeros((n * 114 + 7,), dtype=torch.uint8, device="cuda")
    d_ok = torch.zeros((n,), dtype=torch.uint8, device="cuda")
    ctx = np.frombuffer(b"device ctx", dtype=np.uint8)
    # keygen takes dense rows: the seeds go through a dense copy at an odd offset
    d_s = torch.zeros((n * 57 + 3,), dtype=torch.uint8, device="cuda")
    d_s[3:] = d_seeds[3:].view(n, 59)[:, :57].reshape(-1)
    check(lib().cb200_ed448_keygen(d_s.data_ptr() + 3, d_pk.data_ptr() + 1, d_sk.data_ptr() + 5, n))
    check(lib().cb200_ed448_sign(d_sk.data_ptr() + 5, 114, d_blob.data_ptr(), d_off.data_ptr(), ctx.ctypes.data, len(ctx),
                                 d_sig.data_ptr() + 7, n))
    check(lib().cb200_ed448_verify(d_pk.data_ptr() + 1, 57, d_blob.data_ptr(), d_off.data_ptr(), ctx.ctypes.data, len(ctx),
                                   d_sig.data_ptr() + 7, d_ok.data_ptr(), n))
    torch.cuda.synchronize()
    assert d_ok.sum().item() == n
    s = Ed448()
    pk, sk = s.DeriveKeyBatch(_rows(seeds))
    assert np.array_equal(d_pk[1:].cpu().numpy().reshape(n, 57), pk)
    assert np.array_equal(d_sk[5:].cpu().numpy().reshape(n, 114), sk)
    assert np.array_equal(d_sig[7:].cpu().numpy().reshape(n, 114), s.SignBatch(sk, msgs, b"device ctx"))
    # a shared key at an odd offset, and a misaligned msg_off is refused
    check(lib().cb200_ed448_sign(d_sk.data_ptr() + 5 + 114 * 3, 0, d_blob.data_ptr(), d_off.data_ptr(), None, 0,
                                 d_sig.data_ptr() + 7, n))
    torch.cuda.synchronize()
    assert np.array_equal(d_sig[7:].cpu().numpy().reshape(n, 114), s.SignBatch(s.UnmarshalBinaryPrivateKey(sk[3].tobytes()), msgs))
    assert lib().cb200_ed448_sign(d_sk.data_ptr(), 114, d_blob.data_ptr(), d_off.data_ptr() + 4, None, 0, d_sig.data_ptr(), 1) == -1


def _edd3_reference(seed, msg):
    import oracle
    ex = hashlib.shake_256(seed).digest(89)
    dpk, dsk = oracle.mldsa_keygen(3, ex[:32])
    k = _ossl(ex[32:])
    pk, sk = dpk + k.public_key().public_bytes_raw(), dsk + ex[32:]
    return pk, sk, oracle.mldsa_sign(3, dsk, msg)[0] + k.sign(msg)


def test_eddilithium3_against_oracle_and_rebuilt_reference(cb):
    import oracle
    from circl_b200 import mldsa
    from circl_b200.ed448 import EdDilithium3, ErrContextNotSupported, SignatureOpts
    from oracle import ed448 as oe
    s = EdDilithium3()
    assert (s.PublicKeySize(), s.PrivateKeySize(), s.SignatureSize(), s.SeedSize()) == (2009, 4057, 3407, 57)
    n = 200
    seeds, msgs = _batch(n, 50)
    pk, sk = s.DeriveKeyBatch(_rows(seeds))
    sig = s.SignBatch(sk, msgs)
    for i in range(0, n, 37):
        assert (pk[i].tobytes(), sk[i].tobytes(), sig[i].tobytes()) == _edd3_reference(seeds[i], msgs[i])
        assert (pk[i].tobytes(), sk[i].tobytes()) == oe.eddilithium3_keygen(seeds[i])
        assert sig[i].tobytes() == oe.eddilithium3_sign(sk[i].tobytes(), msgs[i])
    dsig = mldsa.ByName("Dilithium3").SignBatch(np.ascontiguousarray(sk[:, :4000]), msgs)
    assert np.array_equal(dsig, sig[:, :3293])
    assert s.VerifyBatch(pk, msgs, sig).all()
    bad = sig.copy()
    bad[1, 10] ^= 1       # Dilithium3 half
    bad[2, 3300] ^= 1     # Ed448 R
    bad[3, 3406] ^= 1     # Ed448 S, byte 113
    ok = s.VerifyBatch(pk, msgs, bad)
    assert list(np.nonzero(~ok)[0]) == [1, 2, 3]
    assert [oe.eddilithium3_verify(pk[i].tobytes(), msgs[i], bad[i].tobytes()) for i in range(5)] == list(ok[:5])
    assert oracle.mldsa_verify(3, pk[2, :1952].tobytes(), msgs[2], bad[2, :3293].tobytes())
    key = s.UnmarshalBinaryPrivateKey(sk[4].tobytes())
    assert s.Sign(key, b"shared") == _edd3_reference(seeds[4], b"shared")[2]
    shared = s.SignBatch(key, msgs[:16])  # one key for the batch
    assert s.VerifyBatch(s.UnmarshalBinaryPublicKey(pk[4].tobytes()), msgs[:16], shared).all()
    assert not s.Verify(s.UnmarshalBinaryPublicKey(pk[4].tobytes()), b"shared", s.Sign(key, b"shared")[:-1])
    with pytest.raises(ErrContextNotSupported):
        s.Sign(key, b"x", SignatureOpts(b"ctx"))


def test_eddilithium3_device_rows(cb):
    import torch
    from circl_b200._ffi import check, lib
    from circl_b200.ed448 import EdDilithium3
    s = EdDilithium3()
    n = 256
    seeds, msgs = _batch(n, 60)
    blob = np.frombuffer(b"".join(msgs) + b"\0" * 8, dtype=np.uint8)
    off = np.zeros(n + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(m) for m in msgs])
    check(lib().cb200_set_stream(C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    d_seeds = torch.zeros((n * 57 + 1,), dtype=torch.uint8, device="cuda")
    d_seeds[1:] = torch.from_numpy(_rows(seeds).reshape(-1).copy()).cuda()
    d_blob, d_off = torch.from_numpy(blob.copy()).cuda(), torch.from_numpy(off.view(np.int64).copy()).cuda()
    d_pk = torch.zeros((n * 2009 + 3,), dtype=torch.uint8, device="cuda")
    d_sk = torch.zeros((n * 4057 + 5,), dtype=torch.uint8, device="cuda")
    d_sig = torch.zeros((n * 3407 + 7,), dtype=torch.uint8, device="cuda")
    d_st = torch.ones((n,), dtype=torch.uint8, device="cuda")
    d_ok = torch.zeros((n,), dtype=torch.uint8, device="cuda")
    check(lib().cb200_eddilithium3_keygen(d_seeds.data_ptr() + 1, d_pk.data_ptr() + 3, d_sk.data_ptr() + 5, n))
    check(lib().cb200_eddilithium3_sign(d_sk.data_ptr() + 5, 4057, d_blob.data_ptr(), d_off.data_ptr(), d_sig.data_ptr() + 7,
                                        d_st.data_ptr(), n))
    check(lib().cb200_eddilithium3_verify(d_pk.data_ptr() + 3, 2009, d_blob.data_ptr(), d_off.data_ptr(),
                                          d_sig.data_ptr() + 7, d_ok.data_ptr(), n))
    torch.cuda.synchronize()
    assert d_st.sum().item() == 0 and d_ok.sum().item() == n
    pk, sk = s.DeriveKeyBatch(_rows(seeds))
    assert np.array_equal(d_pk[3:].cpu().numpy().reshape(n, 2009), pk)
    assert np.array_equal(d_sk[5:].cpu().numpy().reshape(n, 4057), sk)
    assert np.array_equal(d_sig[7:].cpu().numpy().reshape(n, 3407), s.SignBatch(sk, msgs))


def test_host_batch_split_across_gpus():
    import circl_b200
    from circl_b200 import _ffi
    if _ffi.lib().cb200_device_count() < 2:
        pytest.skip("needs two GPUs")
    circl_b200.init_devices(0)
    try:
        from circl_b200.ed448 import Ed448
        s = Ed448()
        n = (1 << 16) + 11
        seeds, msgs = _batch(n, 70)
        pk, sk = s.DeriveKeyBatch(_rows(seeds))
        sig = s.SignBatch(sk, msgs)
        for i in (0, n // 2 - 1, n // 2, n - 1):
            assert sig[i].tobytes() == _ossl(seeds[i]).sign(msgs[i])
        assert s.VerifyBatch(pk, msgs, sig).all()
    finally:
        circl_b200.shutdown()
