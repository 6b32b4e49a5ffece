"""GPU parity for sign/ed25519 and sign/eddilithium2: the reference's RFC 8032, sign.input and Wycheproof vectors,
OpenSSL's Ed25519 on random batches (shared and per-op keys, host and device pointers), the reference's use of the
private key's public half as given, tampered signatures, and Ed25519-Dilithium2 rebuilt from OpenSSL Ed25519,
hashlib's SHAKE256 and the oracle's round-3 Dilithium2."""
import ctypes as C
import hashlib

import numpy as np
import pytest

from conftest import load_golden

pytestmark = pytest.mark.gpu

L = 2**252 + 27742317777372353535851937790883648493


@pytest.fixture(scope="module")
def cb():
    import circl_b200
    circl_b200.init(0)
    yield circl_b200
    circl_b200.shutdown()


def _rows(items):
    return np.frombuffer(b"".join(items), dtype=np.uint8).reshape(len(items), -1)


def _h(tag, i, n=32):
    return hashlib.shake_256(bytes([tag]) + i.to_bytes(8, "little")).digest(n)


def _ossl(seed):
    from cryptography.hazmat.primitives.asymmetric.ed25519 import Ed25519PrivateKey
    return Ed25519PrivateKey.from_private_bytes(seed)


def _pub(seed):
    return _ossl(seed).public_key().public_bytes_raw()


def test_reference_vectors(cb):
    from circl_b200.eddsa import Ed25519
    v = load_golden("ed25519_vectors.json.gz")
    s = Ed25519()
    kat = v["rfc8032"] + v["sign_input"]
    seeds = _rows([bytes.fromhex(t["seed"]) for t in kat])
    pk, sk = s.DeriveKeyBatch(seeds)
    assert [pk[i].tobytes().hex() for i in range(len(kat))] == [t["pk"] for t in kat]
    msgs = [bytes.fromhex(t["msg"]) for t in kat]
    sig = s.SignBatch(sk, msgs)
    assert [sig[i].tobytes().hex() for i in range(len(kat))] == [t["sig"] for t in kat]
    assert s.VerifyBatch(pk, msgs, sig).all()
    w = v["wycheproof"]
    assert len(w) == 145
    pkw, skw = s.DeriveKeyBatch(_rows([bytes.fromhex(t["seed"]) for t in w]))
    assert all(pkw[i].tobytes().hex() == t["pk"] for i, t in enumerate(w))
    got = []
    for i, t in enumerate(w):
        if t["valid"]:
            assert s.Sign(s.UnmarshalBinaryPrivateKey(skw[i].tobytes()), bytes.fromhex(t["msg"])).hex() == t["sig"]
        got.append(s.Verify(s.UnmarshalBinaryPublicKey(bytes.fromhex(t["pk"])), bytes.fromhex(t["msg"]), bytes.fromhex(t["sig"])))
    assert got == [t["valid"] for t in w]
    full = [i for i, t in enumerate(w) if len(t["sig"]) == 128]  # the same through one batch
    ok = s.VerifyBatch(_rows([bytes.fromhex(w[i]["pk"]) for i in full]), [bytes.fromhex(w[i]["msg"]) for i in full],
                       _rows([bytes.fromhex(w[i]["sig"]) for i in full]))
    assert list(ok) == [w[i]["valid"] for i in full]


def _batch(n, tag):
    lens = [0, 1, 111, 112, 127, 128, 239, 240, 32, 1000]
    seeds = [_h(tag, i) for i in range(n)]
    msgs = [_h(tag + 1, i, lens[i % len(lens)]) if lens[i % len(lens)] else b"" for i in range(n)]
    return seeds, msgs


def test_openssl_parity_per_op_and_shared_keys(cb):
    from circl_b200.eddsa import Ed25519
    s = Ed25519()
    n = 1 << 14
    seeds, msgs = _batch(n, 10)
    msgs[5] = _h(99, 5, 10000)
    pk, sk = s.DeriveKeyBatch(_rows(seeds))
    sig = s.SignBatch(sk, msgs)
    from oracle import ed25519 as oe
    for i in list(range(0, n, 97)) + [5, n - 1]:
        k = _ossl(seeds[i])
        assert pk[i].tobytes() == _pub(seeds[i])
        assert sig[i].tobytes() == k.sign(msgs[i])
    for i in range(0, n, 1601):
        assert (pk[i].tobytes(), sk[i].tobytes()) == oe.ed25519_keygen(seeds[i])
        assert sig[i].tobytes() == oe.ed25519_sign(sk[i].tobytes(), msgs[i])
    assert s.VerifyBatch(pk, msgs, sig).all()
    # one shared key
    key = s.UnmarshalBinaryPrivateKey(sk[7].tobytes())
    sig1 = s.SignBatch(key, msgs[:4096])
    for i in range(0, 4096, 301):
        assert sig1[i].tobytes() == _ossl(seeds[7]).sign(msgs[i])
    assert s.VerifyBatch(s.UnmarshalBinaryPublicKey(pk[7].tobytes()), msgs[:4096], sig1).all()


def test_private_key_public_half_is_used_as_given(cb):
    """ed25519.Sign hashes R || sk[32:64] || M with the second half of the key as given, without recomputing it."""
    from circl_b200.eddsa import Ed25519
    s = Ed25519()
    seed, other = _h(20, 0), _h(20, 1)
    wrong_a = _pub(other)
    sig = s.SignBatch(_rows([seed + wrong_a]), [b"message"])[0].tobytes()
    # the reference's value: R = [r]B with r from SHA-512(prefix || M), k from SHA-512(R || wrong A || M), S = r + k s
    h = hashlib.sha512(seed).digest()
    a = int.from_bytes(h[:32], "little") & ~7 & (2**255 - 1) | 2**254
    r = int.from_bytes(hashlib.sha512(h[32:] + b"message").digest(), "little") % L
    R = _ossl(seed).sign(b"message")[:32]  # R depends on the seed and M only
    k = int.from_bytes(hashlib.sha512(R + wrong_a + b"message").digest(), "little") % L
    assert sig == R + ((r + k * a) % L).to_bytes(32, "little")
    assert sig != _ossl(seed).sign(b"message")
    assert not s.VerifyBatch(_rows([_pub(seed)]), [b"message"], _rows([sig]))[0]


def test_tampered_signatures(cb):
    from circl_b200.eddsa import Ed25519
    s = Ed25519()
    n = 600
    seeds, msgs = _batch(n, 30)
    pk, sk = s.DeriveKeyBatch(_rows(seeds))
    sig = s.SignBatch(sk, msgs).copy()
    pk2, msgs2 = pk.copy(), list(msgs)
    want = np.ones(n, dtype=bool)
    for i in range(0, n, 6):
        kind = (i // 6) % 6
        if kind == 0:
            sig[i, 3] ^= 0x10                      # R
        elif kind == 1:
            sig[i, 40] ^= 0x01                     # S
        elif kind == 2:                            # S + L: same point equation, but not canonical
            S = int.from_bytes(sig[i, 32:].tobytes(), "little") + L
            sig[i, 32:] = np.frombuffer(S.to_bytes(32, "little"), dtype=np.uint8)
        elif kind == 3:
            pk2[i] = np.frombuffer(_pub(_h(31, i)), dtype=np.uint8)  # another key
        elif kind == 4:
            msgs2[i] = msgs2[i] + b"\0"            # message
        else:
            pk2[i, 31] ^= 0x80                     # A with the other sign of x
        want[i] = False
    assert np.array_equal(s.VerifyBatch(pk2, msgs2, sig), want)


def test_device_pointers(cb):
    import torch
    from circl_b200._ffi import check, lib
    from circl_b200.eddsa import Ed25519
    n = 4096
    seeds, msgs = _batch(n, 40)
    blob = np.frombuffer(b"".join(msgs) + b"\0" * 8, dtype=np.uint8)
    off = np.zeros(n + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(m) for m in msgs])
    check(lib().cb200_set_stream(C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    d_seeds = torch.from_numpy(_rows(seeds).copy()).cuda()
    d_blob, d_off = torch.from_numpy(blob.copy()).cuda(), torch.from_numpy(off.view(np.int64).copy()).cuda()
    d_pk = torch.empty((n, 32), dtype=torch.uint8, device="cuda")
    d_sk = torch.empty((n, 64), dtype=torch.uint8, device="cuda")
    d_sig = torch.empty((n, 64), dtype=torch.uint8, device="cuda")
    d_ok = torch.zeros((n,), dtype=torch.uint8, device="cuda")
    check(lib().cb200_ed25519_keygen(d_seeds.data_ptr(), d_pk.data_ptr(), d_sk.data_ptr(), n))
    check(lib().cb200_ed25519_sign(d_sk.data_ptr(), 64, d_blob.data_ptr(), d_off.data_ptr(), d_sig.data_ptr(), n))
    d_sig[9, 0] ^= 1
    check(lib().cb200_ed25519_verify(d_pk.data_ptr(), 32, d_blob.data_ptr(), d_off.data_ptr(), d_sig.data_ptr(),
                                     d_ok.data_ptr(), n))
    torch.cuda.synchronize()
    ok = d_ok.cpu().numpy()
    assert ok.sum() == n - 1 and ok[9] == 0
    d_sig[9, 0] ^= 1
    s = Ed25519()
    pk, sk = s.DeriveKeyBatch(_rows(seeds))
    assert np.array_equal(d_pk.cpu().numpy(), pk) and np.array_equal(d_sk.cpu().numpy(), sk)
    assert np.array_equal(d_sig.cpu().numpy(), s.SignBatch(sk, msgs))
    # rows at the stated 4-byte alignment: keys and signatures inside wider rows at an offset of 4
    rows = torch.zeros((n, 76), dtype=torch.uint8, device="cuda")
    rows[:, 4:68] = d_sk
    out = torch.zeros((n, 72), dtype=torch.uint8, device="cuda")
    check(lib().cb200_ed25519_sign(rows.data_ptr() + 4, 76, d_blob.data_ptr(), d_off.data_ptr(), out.data_ptr() + 4, n))
    torch.cuda.synchronize()
    assert lib().cb200_ed25519_sign(d_sk.data_ptr() + 2, 64, d_blob.data_ptr(), d_off.data_ptr(), out.data_ptr(), 1) == -1
    # the signature output is dense n x 64 starting at out + 4
    flat = out.view(-1)[4:4 + 64 * n].cpu().numpy().reshape(n, 64)
    assert np.array_equal(flat, d_sig.cpu().numpy())


def _edd2_reference(seed, msg):
    import oracle
    ex = hashlib.shake_256(seed).digest(64)
    dpk, dsk = oracle.mldsa_keygen(2, ex[:32])
    pk, sk = dpk + _pub(ex[32:]), dsk + ex[32:]
    sig = oracle.mldsa_sign(2, dsk, msg)[0] + _ossl(ex[32:]).sign(msg)
    return pk, sk, sig


def test_eddilithium2_against_rebuilt_reference(cb):
    import oracle
    from circl_b200 import mldsa
    from circl_b200.eddsa import EdDilithium2
    s = EdDilithium2()
    assert (s.PublicKeySize(), s.PrivateKeySize(), s.SignatureSize(), s.SeedSize()) == (1344, 2560, 2484, 32)
    n = 300
    seeds, msgs = _batch(n, 50)
    pk, sk = s.DeriveKeyBatch(_rows(seeds))
    sig = s.SignBatch(sk, msgs)
    from oracle import ed25519 as oe
    for i in range(0, n, 37):
        assert (pk[i].tobytes(), sk[i].tobytes(), sig[i].tobytes()) == _edd2_reference(seeds[i], msgs[i])
        assert (pk[i].tobytes(), sk[i].tobytes()) == oe.eddilithium2_keygen(seeds[i])  # the project's own oracle
        assert sig[i].tobytes() == oe.eddilithium2_sign(sk[i].tobytes(), msgs[i])
    # the Dilithium2 half is what cb200_mldsa_sign(2, ...) gives for the same key
    dsig = mldsa.ByName("Dilithium2").SignBatch(np.ascontiguousarray(sk[:, :2528]), msgs)
    assert np.array_equal(dsig, sig[:, :2420])
    assert s.VerifyBatch(pk, msgs, sig).all()
    bad = sig.copy()
    bad[1, 10] ^= 1       # Dilithium2 half
    bad[2, 2430] ^= 1     # Ed25519 R
    bad[3, 2483] ^= 1     # Ed25519 S
    ok = s.VerifyBatch(pk, msgs, bad)
    assert list(np.nonzero(~ok)[0]) == [1, 2, 3]
    assert [oe.eddilithium2_verify(pk[i].tobytes(), msgs[i], bad[i].tobytes()) for i in range(6)] == list(ok[:6])
    assert oracle.mldsa_verify(2, pk[2, :1312].tobytes(), msgs[2], bad[2, :2420].tobytes())
    key = s.UnmarshalBinaryPrivateKey(sk[4].tobytes())
    assert s.Sign(key, b"shared") == _edd2_reference(seeds[4], b"shared")[2]
    assert s.Verify(s.UnmarshalBinaryPublicKey(pk[4].tobytes()), b"shared", s.Sign(key, b"shared"))
    assert not s.Verify(s.UnmarshalBinaryPublicKey(pk[4].tobytes()), b"shared", s.Sign(key, b"shared")[:-1])
    from circl_b200.eddsa import ErrContextNotSupported, SignatureOpts
    with pytest.raises(ErrContextNotSupported):
        s.Sign(key, b"x", SignatureOpts(b"ctx"))


def test_eddilithium2_device_rows(cb):
    import torch
    from circl_b200._ffi import check, lib
    from circl_b200.eddsa import EdDilithium2
    s = EdDilithium2()
    n = 512
    seeds, msgs = _batch(n, 60)
    blob = np.frombuffer(b"".join(msgs) + b"\0" * 8, dtype=np.uint8)
    off = np.zeros(n + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(m) for m in msgs])
    check(lib().cb200_set_stream(C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    d_seeds = torch.from_numpy(_rows(seeds).copy()).cuda()
    d_blob, d_off = torch.from_numpy(blob.copy()).cuda(), torch.from_numpy(off.view(np.int64).copy()).cuda()
    d_pk = torch.empty((n, 1344), dtype=torch.uint8, device="cuda")
    d_sk = torch.empty((n, 2560), dtype=torch.uint8, device="cuda")
    sig_rows = torch.zeros((n * 2484 + 4,), dtype=torch.uint8, device="cuda")  # signatures start at byte 4
    d_st = torch.ones((n,), dtype=torch.uint8, device="cuda")
    d_ok = torch.zeros((n,), dtype=torch.uint8, device="cuda")
    check(lib().cb200_eddilithium2_keygen(d_seeds.data_ptr(), d_pk.data_ptr(), d_sk.data_ptr(), n))
    check(lib().cb200_eddilithium2_sign(d_sk.data_ptr(), 2560, d_blob.data_ptr(), d_off.data_ptr(), sig_rows.data_ptr() + 4,
                                        d_st.data_ptr(), n))
    check(lib().cb200_eddilithium2_verify(d_pk.data_ptr(), 1344, d_blob.data_ptr(), d_off.data_ptr(),
                                          sig_rows.data_ptr() + 4, d_ok.data_ptr(), n))
    torch.cuda.synchronize()
    assert d_st.sum().item() == 0 and d_ok.sum().item() == n
    pk, sk = s.DeriveKeyBatch(_rows(seeds))
    assert np.array_equal(d_pk.cpu().numpy(), pk) and np.array_equal(d_sk.cpu().numpy(), sk)
    sig = sig_rows[4:].cpu().numpy().reshape(n, 2484)
    assert np.array_equal(sig, s.SignBatch(sk, msgs))


def test_registry():
    from circl_b200 import eddsa
    assert [s.Name() for s in eddsa.All()] == ["Ed25519", "Ed25519-Dilithium2"]
    assert eddsa.ByName("ED25519-dilithium2").Name() == "Ed25519-Dilithium2"


def test_host_batch_split_across_gpus():
    import circl_b200
    from circl_b200 import _ffi
    if _ffi.lib().cb200_device_count() < 2:
        pytest.skip("needs two GPUs")
    circl_b200.init_devices(0)
    try:
        from circl_b200.eddsa import Ed25519
        s = Ed25519()
        n = 1 << 14
        seeds, msgs = _batch(n, 70)
        pk, sk = s.DeriveKeyBatch(_rows(seeds))
        sig = s.SignBatch(sk, msgs)
        for i in (0, n // 2 - 1, n // 2, n - 1):
            assert sig[i].tobytes() == _ossl(seeds[i]).sign(msgs[i])
        assert s.VerifyBatch(pk, msgs, sig).all()
    finally:
        circl_b200.shutdown()
