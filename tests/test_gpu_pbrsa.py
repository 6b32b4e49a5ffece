"""Partially blind RSA on the GPU against tests/pbrsa_model.py: model parity on 2^12 ops per fixture key with per-op
metadata (empty, 1 byte, lengths around the 128-byte SHA-384 block, 1 KiB), on host buffers and CUDA tensors; edge
rows (0, 1, N - 1, N, N + 1) failing only their own op; keys that fail every op with status 2 (a corrupted qinv, and
primes that are not safe); Verify with wrong, swapped and empty metadata, s >= N and tampered encodings; a round trip
with the model as the client; device rows at odd byte offsets with bad device offsets failing their own op; and host
batches over one staging chunk with a ragged tail, split across GPUs when there are two or more."""
import random

import numpy as np
import pytest

import brsa_model as bm
import pbrsa_model as pm

pytestmark = pytest.mark.gpu
KEYS = ["strong2048", "safe3072", "safe4096", "safe2050", "safe2052", "safe3073", "safe2048u"]


def _metas(rng):
    """16 distinct metadata strings"""
    out = [b"", b"\x01"] + [rng.randbytes(n) for n in (107, 108, 111, 112, 116, 120, 123, 124, 125, 127, 128, 129, 1024)]
    return out + [b"exp=2026-10-18"]


@pytest.fixture(scope="module")
def cb():
    import circl_b200
    circl_b200.init(0)
    yield circl_b200
    circl_b200.shutdown()


@pytest.fixture(scope="module")
def keys():
    return pm.keys()


def _sk(k):
    from circl_b200 import blindrsa
    return blindrsa.PrivateKey(k.n, k.e, k.d, [k.p, k.q])


def _u8(rows):
    return np.frombuffer(b"".join(rows), dtype=np.uint8).reshape(len(rows), -1).copy()


def _dstrings(strings):
    import torch
    off = np.zeros(len(strings) + 1, np.int64)
    np.cumsum([len(m) for m in strings], out=off[1:])
    data = torch.frombuffer(bytearray(b"".join(strings) or b"\0"), dtype=torch.uint8).cuda()
    return data, torch.from_numpy(off).cuda()


@pytest.mark.parametrize("name", KEYS)
def test_blind_sign_matches_the_model(cb, keys, name):
    import torch
    from circl_b200 import partiallyblindrsa as pb
    k = keys[name]
    rng = random.Random(name)
    metas = _metas(rng)
    d = [pm.derive_private(k, m)[1] for m in metas]
    n = 1 << 12
    cs = [rng.randrange(k.n) for _ in range(n)]
    meta = [metas[(i * 7) % 16] for i in range(n)]
    rows = _u8([bm.i2osp(c, k.klen) for c in cs])
    signer = pb.NewSigner(_sk(k))
    sig = signer.BlindSignBatch(rows, meta)  # raises unless every op passed its s^e' mod N == c check
    for i in list(range(0, n, 101)) + list(range(16)) + [n - 1]:
        assert sig[i].tobytes() == bm.i2osp(pow(cs[i], d[(i * 7) % 16], k.n), k.klen), i
    dsig = signer.BlindSignBatch(torch.from_numpy(rows).cuda(), _dstrings(meta))
    assert np.array_equal(dsig.cpu().numpy(), sig)


@pytest.mark.parametrize("name", KEYS)
def test_blind_sign_edge_rows(cb, keys, name):
    from circl_b200 import partiallyblindrsa as pb
    k = keys[name]
    rng = random.Random(name + "edge")
    vals = [rng.randrange(k.n), 0, 1, k.n - 1, k.n, k.n + 1, (1 << (8 * k.klen)) - 1, rng.randrange(k.n)]
    metas = [b"a", b"", b"b" * 200, b"c", b"", b"d", b"", b"e" * 128]
    rows = _u8([bm.i2osp(c, k.klen) for c in vals])
    with pytest.raises(pb.ErrInvalidMessageLength) as ei:
        pb.NewSigner(_sk(k)).BlindSignBatch(rows, metas)
    st, sig = ei.value.status, ei.value.results
    want = [pm.blind_sign(k, bm.i2osp(c, k.klen), m) for c, m in zip(vals, metas)]
    assert list(st) == [w[0] for w in want] == [0, 0, 0, 0, 2, 1, 1, 0]
    assert [sig[i].tobytes() for i in range(len(vals))] == [w[1] for w in want]
    signer = pb.NewSigner(_sk(k))
    with pytest.raises(pb.ErrInternal):
        signer.BlindSign(bm.i2osp(k.n, k.klen), b"m")
    with pytest.raises(pb.ErrUnexpectedSize):
        signer.BlindSignBatch(rows, metas[:-1])


def _raw_sign(L, k, p, q, qinv, rows, metas):
    n = rows.shape[0]
    off = np.zeros(n + 1, np.uint64)
    np.cumsum([len(m) for m in metas], out=off[1:])
    mb = np.frombuffer(b"".join(metas) or b"\0", np.uint8).copy()
    sig, st = np.full((n, k.klen), 0x5a, np.uint8), np.full(n, 9, np.uint8)
    f = [bm.i2osp(v, (v.bit_length() + 7) // 8 or 1) for v in (k.n, p, q, qinv)]
    from circl_b200 import _ffi
    _ffi.check(L.cb200_pbrsa_blind_sign(f[0], len(f[0]), f[1], len(f[1]), f[2], len(f[2]), f[3], len(f[3]),
                                        rows.ctypes.data, mb.ctypes.data, off.ctypes.data, sig.ctypes.data,
                                        st.ctypes.data, n))
    return st, sig


@pytest.mark.parametrize("name", ["strong2048", "safe4096", "safe2048u"])
def test_corrupted_qinv_fails_every_op(cb, keys, name):
    from circl_b200 import _ffi
    k = keys[name]
    rng = random.Random(name + "qinv")
    rows = _u8([bm.i2osp(rng.randrange(2, k.n - 1), k.klen) for _ in range(256)])
    metas = [bytes([i]) * (i % 5) for i in range(256)]
    qinv = pow(k.q, -1, k.p) ^ 8
    st, sig = _raw_sign(_ffi.lib(), k, k.p, k.q, qinv, rows, metas)
    assert (st == 2).all() and not sig.any()


def test_key_whose_primes_are_not_safe_fails_every_op(cb):
    from circl_b200 import _ffi, partiallyblindrsa as pb
    w = bm.all_keys()["rsa2048u"]  # primes = 3 mod 4 whose halves are composite: NewSigner refuses it
    with pytest.raises(pb.ErrInvalidPrivateKey):
        pb.NewSigner(_sk(w))
    rng = random.Random(3)
    rows = _u8([bm.i2osp(rng.randrange(2, w.n - 1), w.klen) for _ in range(256)])
    st, sig = _raw_sign(_ffi.lib(), w, w.p, w.q, pow(w.q, -1, w.p), rows, [b"m"] * 256)
    assert (st == 2).all() and not sig.any()


@pytest.mark.parametrize("name", KEYS)
def test_verify(cb, keys, name):
    import torch
    from circl_b200 import partiallyblindrsa as pb
    from circl_b200._ffi import Cb200Error
    k = keys[name]
    rng = random.Random(name + "verify")
    metas = _metas(rng)
    msgs, meta, sigs, want = [], [], [], []
    for i, md in enumerate(metas):
        msg = rng.randbytes(rng.randrange(0, 300))
        sig = pm.sign(k, msg, md, rng)
        bad = bytearray(sig)
        bad[k.klen // 2] ^= 0x10
        cases = [(msg, md, sig), (msg, md + b"\0", sig), (msg, metas[(i + 1) % 16], sig), (msg + b"\0", md, sig),
                 (msg, md, bytes(bad)), (msg, md, bm.i2osp(k.n, k.klen)), (msg, md, bm.i2osp(k.n + 1, k.klen))]
        for m, mt, s in cases:
            msgs.append(m), meta.append(mt), sigs.append(s), want.append(pm.verify_status(k, m, mt, s))
    # a valid encoding under the key of one metadata string, signed for another (the e' of the first)
    e0, d0 = pm.derive_private(k, metas[0])
    em = bm.emsa_pss_encode(pm.frame(b"x", metas[1]), k.n.bit_length() - 1, rng.randbytes(48))
    s = bm.i2osp(pow(bm.os2ip(em), d0, k.n), k.klen)
    msgs.append(b"x"), meta.append(metas[1]), sigs.append(s), want.append(2)
    msgs.append(b"x"), meta.append(metas[0]), sigs.append(s), want.append(2)
    assert want.count(0) == 16 and want.count(1) == 32
    v = pb.NewVerifier(_sk(k).PublicKey)
    with pytest.raises(pb.ErrVerification) as ei:
        v.VerifyBatch(msgs, meta, _u8(sigs))
    assert list(ei.value.status) == want
    with pytest.raises(pb.ErrVerification) as ei:
        v.VerifyBatch(_dstrings(msgs), _dstrings(meta), torch.from_numpy(_u8(sigs)).cuda())
    assert ei.value.status.cpu().tolist() == want
    with pytest.raises(Cb200Error):  # CUDA messages with host metadata
        v.VerifyBatch(_dstrings(msgs), meta, torch.from_numpy(_u8(sigs)).cuda())
    good = [i for i, x in enumerate(want) if x == 0]
    v.VerifyBatch([msgs[i] for i in good], [meta[i] for i in good], _u8([sigs[i] for i in good]))
    v.Verify(msgs[good[0]], meta[good[0]], sigs[good[0]])
    with pytest.raises(pb.ErrVerification):
        v.Verify(msgs[good[0]], meta[good[0]], sigs[good[0]][1:])


@pytest.mark.parametrize("name", KEYS)
def test_round_trip_with_the_model_client(cb, keys, name):
    from circl_b200 import partiallyblindrsa as pb
    k = keys[name]
    rng = random.Random(name + "rt")
    metas = _metas(rng)
    msgs, blinded, invs = [], [], []
    for md in metas:
        m = rng.randbytes(rng.randrange(300))
        b, inv = pm.blind(k, m, md, rng.randbytes(48), rng.randrange(2, k.n - 1))
        msgs.append(m), blinded.append(b), invs.append(inv)
    bsig = pb.NewSigner(_sk(k)).BlindSignBatch(_u8(blinded), metas)
    sigs = [pm.finalize(k, m, md, bsig[i].tobytes(), invs[i]) for i, (m, md) in enumerate(zip(msgs, metas))]
    pb.NewVerifier(_sk(k).PublicKey).VerifyBatch(msgs, metas, _u8(sigs))


def test_device_rows_at_odd_offsets(cb, keys):
    import torch
    from circl_b200 import _ffi
    L = _ffi.lib()
    k = keys["safe3073"]
    rng = random.Random(5)
    n = 67
    cs = [rng.randrange(k.n) for _ in range(n)]
    metas = [rng.randbytes(i % 40) for i in range(n)]
    rows = _u8([bm.i2osp(c, k.klen) for c in cs])
    f = [bm.i2osp(v, (v.bit_length() + 7) // 8) for v in (k.n, k.p, k.q, pow(k.q, -1, k.p))]
    key = [f[0], len(f[0]), f[1], len(f[1]), f[2], len(f[2]), f[3], len(f[3])]
    buf = torch.zeros(n * k.klen + 3, dtype=torch.uint8, device="cuda")
    buf[1:1 + n * k.klen] = torch.from_numpy(rows.reshape(-1)).cuda()
    mb = b"".join(metas)
    dmeta = torch.zeros(len(mb) + 2, dtype=torch.uint8, device="cuda")
    dmeta[1:1 + len(mb)] = torch.frombuffer(bytearray(mb), dtype=torch.uint8).cuda()
    off = np.zeros(n + 1, np.int64)
    np.cumsum([len(m) for m in metas], out=off[1:])
    off[10] = off[9] - 1  # op 9's offsets decrease; op 10 then starts one byte early, a metadata string of its own
    doff = torch.from_numpy(off).cuda()
    out = torch.full((n * k.klen + 5,), 0x77, dtype=torch.uint8, device="cuda")
    st = torch.full((n + 3,), 9, dtype=torch.uint8, device="cuda")
    _ffi.check(L.cb200_set_stream(torch.cuda.current_stream().cuda_stream))
    _ffi.check(L.cb200_pbrsa_blind_sign(*key, buf.data_ptr() + 1, dmeta.data_ptr() + 1, doff.data_ptr(),
                                        out.data_ptr() + 3, st.data_ptr() + 1, n))
    torch.cuda.synchronize()
    o = out.cpu().numpy()
    stl = st.cpu().tolist()
    assert stl[0] == 9 and stl[n + 1:] == [9, 9]
    assert o[:3].tolist() == [0x77] * 3 and o[3 + n * k.klen:].tolist() == [0x77, 0x77]
    sigs = o[3:3 + n * k.klen].reshape(n, k.klen)
    for i in range(n):
        if i == 9:
            assert stl[1 + i] == 2 and not sigs[i].any()
            continue
        md = mb[off[i]:off[i + 1]]
        assert stl[1 + i] == 0, i
        if i % 7 == 0 or i == 10:
            assert sigs[i].tobytes() == pm.blind_sign(k, bm.i2osp(cs[i], k.klen), md)[1], i
    # Verify: messages, metadata and signatures at odd offsets; one op with decreasing metadata offsets, one s = N
    msgs = [rng.randbytes(rng.randrange(200)) for _ in range(n)]
    metas = [rng.randbytes(i % 50) for i in range(n)]
    sv = [pm.sign(k, m, md, rng) if i % 9 == 0 else bytes(k.klen) for i, (m, md) in enumerate(zip(msgs, metas))]
    sv[18] = bm.i2osp(k.n, k.klen)
    want = [pm.verify_status(k, m, md, s) for m, md, s in zip(msgs, metas, sv)]
    want[27] = 2
    dm, dmo = _dstrings([b"?" + msgs[0]] + msgs[1:])
    dmd, dmdo = _dstrings(metas)
    dmdo[28] = dmdo[27] - 1  # op 27 (a valid signature) has metadata offsets that decrease
    dmo[0] = 1
    dsig = torch.zeros(n * k.klen + 1, dtype=torch.uint8, device="cuda")
    dsig[1:] = torch.from_numpy(_u8(sv).reshape(-1)).cuda()
    st = torch.full((n + 1,), 9, dtype=torch.uint8, device="cuda")
    f0 = f[0]
    _ffi.check(L.cb200_pbrsa_verify(f0, len(f0), dm.data_ptr(), dmo.data_ptr(), dmd.data_ptr(), dmdo.data_ptr(),
                                    dsig.data_ptr() + 1, st.data_ptr() + 1, n))
    torch.cuda.synchronize()
    assert st.cpu().tolist() == [9] + want
    assert want.count(0) >= 6


def test_host_batch_over_a_staging_chunk_and_across_gpus(keys):
    import circl_b200
    from circl_b200 import partiallyblindrsa as pb
    circl_b200.init_devices(0)  # every visible GPU; with one, the batch still crosses a staging chunk
    try:
        k = keys["strong2048"]
        rng = random.Random(77)
        metas = _metas(rng)
        d = [pm.derive_private(k, m)[1] for m in metas]
        n = (1 << 14) + 5
        cs = np.frombuffer(rng.randbytes(n * k.klen), np.uint8).reshape(n, k.klen).copy()
        cs[:, 0] &= 0x7f  # below N (whose top byte is at least 0x80)
        meta = [metas[i % 16] for i in range(n)]
        sig = pb.NewSigner(_sk(k)).BlindSignBatch(cs, meta)
        for i in list(range(0, n, 1531)) + [n - 1, (1 << 14) - 1, 1 << 14, (1 << 14) + 1]:
            assert sig[i].tobytes() == bm.i2osp(pow(bm.os2ip(cs[i].tobytes()), d[i % 16], k.n), k.klen), i
        # Verify across the same chunks: 64 signatures repeated, one broken near the chunk edge
        msgs64 = [rng.randbytes(rng.randrange(100)) for _ in range(64)]
        sig64 = [pm.sign(k, msgs64[j], metas[j % 16], rng) for j in range(64)]
        msgs = [msgs64[i % 64] for i in range(n)]
        meta = [metas[(i % 64) % 16] for i in range(n)]
        sigs = _u8([sig64[i % 64] for i in range(n)])
        edge = (1 << 14) + 2
        meta[edge] = meta[edge] + b"!"
        with pytest.raises(pb.ErrVerification) as ei:
            pb.NewVerifier(_sk(k).PublicKey).VerifyBatch(msgs, meta, sigs)
        st = ei.value.status
        assert st[edge] == 2 and int((st != 0).sum()) == 1
    finally:
        circl_b200.shutdown()
