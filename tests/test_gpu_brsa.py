"""RSA blind signatures on the GPU against the RFC 9474 vectors, tests/brsa_model.py and OpenSSL: the four vectors
through the C ABI; model parity on 2^12 random blinded messages under every fixture key, on host buffers and CUDA
tensors; edge rows (0, 1, N - 1, N, N + 1) failing only their own op; Verify with one tampered row per EMSA-PSS failure
class and a signature under the other salt length; empty and multi-block messages; a key with a corrupted dp; a full
round trip with the model as the client; device rows at odd byte offsets; and a host batch split across GPUs."""
import random

import numpy as np
import pytest

import brsa_model as bm

pytestmark = pytest.mark.gpu
KEYS = ["rsa2048", "rsa3072", "rsa3073", "rsa2048e3", "rsa2048u", "rsa3000u", "rsa4096"]


@pytest.fixture(scope="module")
def cb():
    import circl_b200
    circl_b200.init(0)
    yield circl_b200
    circl_b200.shutdown()


@pytest.fixture(scope="module")
def keys():
    return bm.all_keys()


def _sk(k):
    from circl_b200 import blindrsa
    return blindrsa.PrivateKey(k.n, k.e, k.d, [k.p, k.q])


def _pk(k):
    from circl_b200 import blindrsa
    return blindrsa.PublicKey(k.n, k.e)


def _u8(rows):
    return np.frombuffer(b"".join(rows), dtype=np.uint8).reshape(len(rows), -1).copy()


def _x(h):
    return bytes.fromhex(h)


def test_rfc9474_vectors_through_the_c_abi(cb):
    from circl_b200 import _ffi
    L = _ffi.lib()
    k = bm.rfc_key()
    dp, dq, qinv = k.crt()
    fields = [bm.i2osp(v, (v.bit_length() + 7) // 8) for v in (k.n, k.e, k.p, k.q, dp, dq, qinv)]
    args = []
    for f in fields:
        args += [f, len(f)]
    for variant, v in enumerate(bm.rfc_vectors()):
        blinded = np.frombuffer(_x(v["blinded_msg"]), np.uint8).copy()
        sig, st = np.zeros(k.klen, np.uint8), np.ones(1, np.uint8)
        _ffi.check(L.cb200_brsa_blind_sign(*args, blinded.ctypes.data, sig.ctypes.data, st.ctypes.data, 1))
        assert st[0] == 0 and sig.tobytes().hex() == v["blind_sig"]
        msg = np.frombuffer(_x(v["input_msg"]), np.uint8).copy()
        off = np.array([0, len(msg)], np.uint64)
        s = np.frombuffer(_x(v["sig"]), np.uint8).copy()
        _ffi.check(L.cb200_brsa_verify(variant, fields[0], len(fields[0]), fields[1], len(fields[1]), msg.ctypes.data,
                                       off.ctypes.data, s.ctypes.data, st.ctypes.data, 1))
        assert st[0] == 0


@pytest.mark.parametrize("name", KEYS)
def test_blind_sign_matches_the_model(cb, keys, name):
    import torch
    from circl_b200 import blindrsa
    k = keys[name]
    rng = random.Random(name)
    n = 1 << 12
    cs = [rng.randrange(k.n) for _ in range(n)]
    rows = _u8([bm.i2osp(c, k.klen) for c in cs])
    signer = blindrsa.NewSigner(_sk(k))
    sig = signer.BlindSignBatch(rows)
    dp, dq, qinv = k.crt()
    for i in list(range(0, n, 97)) + [n - 1]:  # the model is pure Python: a stride sample plus every check below
        assert sig[i].tobytes() == bm.i2osp(pow(cs[i], k.d, k.n), k.klen), i
    # every row: s^e mod N == c
    assert all(pow(bm.os2ip(sig[i].tobytes()), k.e, k.n) == cs[i] for i in range(n))
    dsig = signer.BlindSignBatch(torch.from_numpy(rows).cuda())
    assert np.array_equal(dsig.cpu().numpy(), sig)


@pytest.mark.parametrize("name", KEYS)
def test_blind_sign_edge_rows(cb, keys, name):
    from circl_b200 import blindrsa
    k = keys[name]
    rng = random.Random(name + "edge")
    vals = [rng.randrange(k.n), 0, 1, k.n - 1, k.n, k.n + 1, (1 << (8 * k.klen)) - 1, rng.randrange(k.n)]
    rows = _u8([bm.i2osp(c, k.klen) for c in vals])
    with pytest.raises(blindrsa.ErrInvalidMessageLength) as ei:
        blindrsa.NewSigner(_sk(k)).BlindSignBatch(rows)
    st, sig = ei.value.status, ei.value.results
    want = [bm.blind_sign(k, bm.i2osp(c, k.klen)) for c in vals]
    assert list(st) == [w[0] for w in want] == [0, 0, 0, 0, 2, 1, 1, 0]
    assert [sig[i].tobytes() for i in range(len(vals))] == [w[1] for w in want]
    assert sig[1].tobytes() == bytes(k.klen)  # c = 0 signs to zero
    signer = blindrsa.NewSigner(_sk(k))
    with pytest.raises(blindrsa.ErrInternal):
        signer.BlindSign(bm.i2osp(k.n, k.klen))
    with pytest.raises(blindrsa.ErrUnexpectedSize):
        signer.BlindSign(bytes(k.klen - 1))
    with pytest.raises(blindrsa.ErrUnexpectedSize):
        signer.BlindSignBatch(np.zeros((2, k.klen + 1), np.uint8))


@pytest.mark.parametrize("name", KEYS)
def test_corrupted_dp_fails_every_op(cb, keys, name):
    from circl_b200 import blindrsa
    k = keys[name]
    sk = _sk(k)
    signer = blindrsa.NewSigner(sk)
    f = list(signer._fields)
    f[4] = bm.i2osp(bm.os2ip(f[4]) ^ 4, len(f[4]))
    signer._fields = f
    rng = random.Random(name + "dp")
    rows = _u8([bm.i2osp(rng.randrange(2, k.n - 1), k.klen) for _ in range(256)])
    with pytest.raises(blindrsa.ErrInternal) as ei:
        signer.BlindSignBatch(rows)
    assert (ei.value.status == 2).all() and not ei.value.results.any()


@pytest.mark.parametrize("name", KEYS)
def test_verify_failure_classes(cb, keys, name):
    import torch
    from circl_b200 import blindrsa
    k = keys[name]
    rng = random.Random(name + "verify")
    for variant in range(4):
        slen = bm.VARIANTS[variant][1]
        msgs, sigs, want = [], [], []
        for msg in (b"", b"x", rng.randbytes(111), rng.randbytes(112), rng.randbytes(128), rng.randbytes(1000)):
            cases = bm.tampered(k, slen, msg, rng)
            for _, s, st in cases:
                msgs.append(msg), sigs.append(s), want.append(st)
            other = bm.tampered(k, 48 - slen, msg, rng)[0][1]  # valid under the other salt length
            msgs.append(msg), sigs.append(other), want.append(2)
        v = blindrsa.NewVerifier(variant, _pk(k))
        with pytest.raises(blindrsa.ErrVerification) as ei:
            v.VerifyBatch(msgs, _u8(sigs))
        assert list(ei.value.status) == want
        # the same batch on CUDA tensors
        off = np.zeros(len(msgs) + 1, np.int64)
        np.cumsum([len(m) for m in msgs], out=off[1:])
        dm = torch.frombuffer(bytearray(b"".join(msgs)), dtype=torch.uint8).cuda()
        with pytest.raises(blindrsa.ErrVerification) as ei:
            v.VerifyBatch((dm, torch.from_numpy(off).cuda()), torch.from_numpy(_u8(sigs)).cuda())
        assert ei.value.status.cpu().tolist() == want
        from circl_b200._ffi import Cb200Error
        with pytest.raises(Cb200Error) as ei:  # CUDA messages with host signatures: an argument error, not a key error
            v.VerifyBatch((dm, torch.from_numpy(off).cuda()), _u8(sigs))
        assert not isinstance(ei.value, blindrsa.ErrInvalidKey) and ei.value.code == -1
        good = [i for i, w in enumerate(want) if w == 0]
        v.VerifyBatch([msgs[i] for i in good], _u8([sigs[i] for i in good]))
        v.Verify(msgs[good[0]], sigs[good[0]])
        with pytest.raises(blindrsa.ErrVerification):
            v.Verify(msgs[good[0]], sigs[good[0]][1:])


@pytest.mark.parametrize("name", KEYS)
def test_round_trip_with_the_model_client(cb, keys, name):
    from circl_b200 import blindrsa
    from cryptography.hazmat.primitives import hashes
    from cryptography.hazmat.primitives.asymmetric import padding, rsa
    k = keys[name]
    rng = random.Random(name + "rt")
    ossl = rsa.RSAPublicNumbers(k.e, k.n).public_key()
    for variant in range(4):
        _, slen, plen = bm.VARIANTS[variant]
        prepared, blinded, invs = [], [], []
        for i in range(8):
            p = bm.prepare(variant, rng.randbytes(rng.randrange(300)), rng.randbytes(32))
            b, inv = bm.blind(k, variant, p, rng.randbytes(slen), rng.randrange(2, k.n - 1))
            prepared.append(p), blinded.append(b), invs.append(inv)
        bsig = blindrsa.NewSigner(_sk(k)).BlindSignBatch(_u8(blinded))
        sigs = [bm.finalize(k, variant, p, bsig[i].tobytes(), invs[i]) for i, p in enumerate(prepared)]
        blindrsa.NewVerifier(variant, _pk(k)).VerifyBatch(prepared, _u8(sigs))
        for p, s in zip(prepared, sigs):
            ossl.verify(s, p, padding.PSS(padding.MGF1(hashes.SHA384()), slen), hashes.SHA384())


def test_device_rows_at_odd_offsets(cb, keys):
    import torch
    from circl_b200 import _ffi
    L = _ffi.lib()
    k = keys["rsa3073"]
    rng = random.Random(5)
    n = 67
    cs = [rng.randrange(k.n) for _ in range(n)]
    rows = _u8([bm.i2osp(c, k.klen) for c in cs])
    dp, dq, qinv = k.crt()
    fields = [bm.i2osp(v, (v.bit_length() + 7) // 8) for v in (k.n, k.e, k.p, k.q, dp, dq, qinv)]
    args = []
    for f in fields:
        args += [f, len(f)]
    buf = torch.zeros(n * k.klen + 3, dtype=torch.uint8, device="cuda")
    buf[1:1 + n * k.klen] = torch.from_numpy(rows.reshape(-1)).cuda()
    out = torch.zeros(n * k.klen + 5, dtype=torch.uint8, device="cuda")
    st = torch.full((n + 3,), 9, dtype=torch.uint8, device="cuda")
    _ffi.check(L.cb200_set_stream(torch.cuda.current_stream().cuda_stream))
    _ffi.check(L.cb200_brsa_blind_sign(*args, buf.data_ptr() + 1, out.data_ptr() + 3, st.data_ptr() + 1, n))
    torch.cuda.synchronize()
    o = out.cpu().numpy()
    assert st.cpu().tolist() == [9] + [0] * n + [9, 9]
    assert o[:3].tolist() == [0, 0, 0]
    sigs = o[3:3 + n * k.klen].reshape(n, k.klen)
    assert all(sigs[i].tobytes() == bm.i2osp(pow(cs[i], k.d, k.n), k.klen) for i in range(0, n, 11))
    # Verify: messages and signatures at odd offsets
    msgs = [rng.randbytes(rng.randrange(200)) for _ in range(n)]
    sv = _u8([bm.raw_sign(k, bm.os2ip(bm.emsa_pss_encode(m, k.n.bit_length() - 1, b""))) for m in msgs])
    sv[7] = np.frombuffer(bm.i2osp(k.n, k.klen), np.uint8)
    mb = b"".join(msgs)
    dmsg = torch.zeros(len(mb) + 1, dtype=torch.uint8, device="cuda")
    dmsg[1:] = torch.frombuffer(bytearray(mb), dtype=torch.uint8).cuda()
    off = np.zeros(n + 1, np.int64)
    np.cumsum([len(m) for m in msgs], out=off[1:])
    doff = torch.from_numpy(off).cuda()
    dsig = torch.zeros(n * k.klen + 1, dtype=torch.uint8, device="cuda")
    dsig[1:] = torch.from_numpy(sv.reshape(-1)).cuda()
    st = torch.full((n + 1,), 9, dtype=torch.uint8, device="cuda")
    _ffi.check(L.cb200_brsa_verify(3, fields[0], len(fields[0]), fields[1], len(fields[1]), dmsg.data_ptr() + 1,
                                   doff.data_ptr(), dsig.data_ptr() + 1, st.data_ptr() + 1, n))
    torch.cuda.synchronize()
    assert st.cpu().tolist() == [9] + [1 if i == 7 else 0 for i in range(n)]


def test_status_is_required(cb, keys):
    from circl_b200 import _ffi
    k = keys["rsa2048"]
    L = _ffi.lib()
    dp, dq, qinv = k.crt()
    args = []
    for v in (k.n, k.e, k.p, k.q, dp, dq, qinv):
        f = bm.i2osp(v, (v.bit_length() + 7) // 8)
        args += [f, len(f)]
    z = np.zeros(k.klen, np.uint8)
    assert L.cb200_brsa_blind_sign(*args, z.ctypes.data, z.ctypes.data, None, 1) == -1


def test_host_batch_split_across_gpus(keys):
    import circl_b200
    from circl_b200 import blindrsa
    circl_b200.init_devices(0)  # every visible GPU; with one, the batch still crosses staging chunks
    try:
        k = keys["rsa2048"]
        rng = random.Random(77)
        n = 3 * (1 << 14) + 5  # several staging chunks and, with more than one GPU, several shards
        cs = np.frombuffer(rng.randbytes(n * k.klen), np.uint8).reshape(n, k.klen).copy()
        cs[:, 0] &= 0x7f  # below N (whose top byte is at least 0x80)
        sig = blindrsa.NewSigner(_sk(k)).BlindSignBatch(cs)
        for i in list(range(0, n, 4099)) + [n - 1, (1 << 14) - 1, 1 << 14]:
            assert sig[i].tobytes() == bm.i2osp(pow(bm.os2ip(cs[i].tobytes()), k.d, k.n), k.klen), i
        msgs = [bytes([i & 255]) * (i % 300) for i in range(n)]
        # signatures of the deterministic PSSZero encoding, built by the GPU from the model's encodings
        ems = np.frombuffer(b"".join(bm.emsa_pss_encode(m, k.n.bit_length() - 1, b"") for m in msgs[:512]),
                            np.uint8).reshape(512, -1)
        ems = np.concatenate([np.zeros((512, k.klen - ems.shape[1]), np.uint8), ems], axis=1)
        s512 = blindrsa.NewSigner(_sk(k)).BlindSignBatch(ems)
        reps = (n + 511) // 512
        sigs = np.concatenate([s512] * reps)[:n]
        msgs = [msgs[i % 512] for i in range(n)]
        blindrsa.NewVerifier(3, _pk(k)).VerifyBatch(msgs, sigs)
    finally:
        circl_b200.shutdown()
