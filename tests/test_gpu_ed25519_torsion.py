"""GPU: Ed25519 and Ed25519-Dilithium2 verification on small-order and mixed-order keys and on non-canonical S, A and R
encodings, every verdict from the Python-integer model of the reference's cofactorless rule (tests/ed25519_model.py),
which the CPU suite checks against the oracle, OpenSSL and the host build of ed25519.cuh.  Per-op keys on host buffers,
rows inside wider CUDA tensors, one shared key per low-order point, signing under mixed-order keys used as given, and
the composite with either half failing."""
import ctypes as C
import hashlib
import random

import numpy as np
import pytest

import ed25519_model as M

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cb():
    import circl_b200
    circl_b200.init(0)
    yield circl_b200
    circl_b200.shutdown()


@pytest.fixture(scope="module")
def cases():
    return M.torsion_cases()


def _rows(items):
    return np.frombuffer(b"".join(items), dtype=np.uint8).reshape(len(items), -1)


def _names_of_mismatches(cases, got):
    return [c[0] for c, g in zip(cases, got) if bool(g) != c[4]]


def _ossl_batch(n, tag):
    """n valid (pk, msg, sig) from OpenSSL under n keys."""
    from cryptography.hazmat.primitives.asymmetric.ed25519 import Ed25519PrivateKey
    out = []
    for i in range(n):
        seed = hashlib.shake_256(bytes([tag]) + i.to_bytes(4, "little")).digest(32)
        msg = hashlib.shake_256(bytes([tag + 1]) + i.to_bytes(4, "little")).digest(i % 300)
        k = Ed25519PrivateKey.from_private_bytes(seed)
        out.append((k.public_key().public_bytes_raw(), msg, k.sign(msg)))
    return out


def test_every_case_per_op_keys(cb, cases):
    """All cases in one batch, then the same cases at random positions among 4096 valid signatures."""
    from circl_b200.eddsa import Ed25519
    s = Ed25519()
    ok = s.VerifyBatch(_rows([c[1] for c in cases]), [c[2] for c in cases], _rows([c[3] for c in cases]))
    assert not _names_of_mismatches(cases, ok)
    valid = _ossl_batch(4096, 80)
    n = len(valid) + len(cases)
    where = random.Random(1).sample(range(n), len(cases))
    ops = [(pk, msg, sig, True) for pk, msg, sig in valid]
    for pos, c in sorted(zip(where, cases)):
        ops.insert(pos, (c[1], c[2], c[3], c[4]))
    ok = s.VerifyBatch(_rows([o[0] for o in ops]), [o[1] for o in ops], _rows([o[2] for o in ops]))
    assert np.array_equal(ok, np.array([o[3] for o in ops])), np.nonzero(ok != np.array([o[3] for o in ops]))


def test_every_case_device_rows(cb, cases):
    """cb200_ed25519_verify on CUDA tensors: keys at byte 4 of 40-byte rows, signatures and messages starting at byte
    4 of their buffers, each op next to a valid one."""
    import torch
    from circl_b200._ffi import check, lib
    valid = _ossl_batch(len(cases), 81)
    ops = [o for c, v in zip(cases, valid) for o in ((c[1], c[2], c[3], c[4]), v + (True,))]
    n = len(ops)
    keys = np.zeros((n, 40), dtype=np.uint8)
    keys[:, 4:36] = _rows([o[0] for o in ops])
    sigs = np.frombuffer(b"\0" * 4 + b"".join(o[2] for o in ops), dtype=np.uint8)
    blob = np.frombuffer(b"\0" * 4 + b"".join(o[1] for o in ops) + b"\0" * 8, dtype=np.uint8)
    off = np.zeros(n + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(o[1]) for o in ops])
    check(lib().cb200_set_stream(C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    d_keys, d_sigs = torch.from_numpy(keys).cuda(), torch.from_numpy(sigs.copy()).cuda()
    d_blob, d_off = torch.from_numpy(blob.copy()).cuda(), torch.from_numpy(off.view(np.int64).copy()).cuda()
    d_ok = torch.full((n,), 7, dtype=torch.uint8, device="cuda")
    check(lib().cb200_ed25519_verify(d_keys.data_ptr() + 4, 40, d_blob.data_ptr() + 4, d_off.data_ptr(),
                                     d_sigs.data_ptr() + 4, d_ok.data_ptr(), n))
    torch.cuda.synchronize()
    assert d_ok.cpu().numpy().tolist() == [int(o[3]) for o in ops]


def test_shared_low_order_keys(cb):
    """Each point of order dividing 8 as one PublicKey (stride 0) under 264 signatures R = encode([S mod L] B), S at
    the edges and beyond L: the verdict is S < L and [k] T = O, and the model agrees on every eighth op."""
    from circl_b200.eddsa import Ed25519
    s = Ed25519()
    rng = random.Random(2)
    svals = [0, 1, 2, M.L - 1, 2**252, M.L, M.L + 1, 2**256 - 1] + [rng.randrange(M.L) for _ in range(3)]
    R = {S: M.encode(M.mul_base(S % M.L)) for S in svals}
    for j, T in enumerate(M.TORSION):
        A, n = M.encode(T), M.ORDERS[j]
        msgs = [b"shared %d %d" % (j, i) for i in range(264)]
        sigs = [R[S] + S.to_bytes(32, "little") for S in (svals[i % len(svals)] for i in range(264))]
        want = [int.from_bytes(sg[32:], "little") < M.L and M.sha512_mod_l(sg[:32], A, m) % n == 0
                for m, sg in zip(msgs, sigs)]
        assert all(M.verify(A, msgs[i], sigs[i]) == want[i] for i in range(0, 264, 8))
        assert set(want) == {True, False}
        ok = s.VerifyBatch(s.UnmarshalBinaryPublicKey(A), msgs, _rows(sigs))
        assert ok.tolist() == want, j


def test_sign_under_mixed_order_keys(cb):
    """seed || encode([a] B + T) for T of order 2, 4 and 8, 512 messages each: the device's signatures are the model's,
    and its verdicts (true iff ord(T) divides k) are the model's."""
    from circl_b200.eddsa import Ed25519
    s = Ed25519()
    sks, pks, msgs = [], [], []
    for n, T in ((2, M.T2), (4, M.T4), (8, M.T8)):
        seed = hashlib.sha512(b"mixed-order %d" % n).digest()[:32]
        A = M.encode(M.add(M.mul_base(M.expand(seed)[0]), T))
        for i in range(512):
            sks.append(seed + A)
            pks.append(A)
            msgs.append(b"mixed-order %d, %d" % (n, i))
    sig = s.SignBatch(_rows(sks), msgs)
    want_sig = [M.sign(sk[:32], sk[32:], m) for sk, m in zip(sks, msgs)]
    assert [sig[i].tobytes() for i in range(len(msgs))] == want_sig
    for t, n in enumerate((2, 4, 8)):
        ks = {M.sha512_mod_l(want_sig[i][:32], pks[i], msgs[i]) % 8 for i in range(512 * t, 512 * (t + 1))}
        assert ks == set(range(8))
    want = [M.verify(A, m, sg) for A, m, sg in zip(pks, msgs, want_sig)]
    assert set(want[:512]) == set(want[512:1024]) == set(want[1024:]) == {True, False}
    assert s.VerifyBatch(_rows(pks), msgs, sig).tolist() == want


def test_eddilithium2_cases(cb, cases):
    """A valid Dilithium2 half from the oracle joined to each case gives the model's verdict on the Ed25519 half; a
    corrupted Dilithium2 half under a valid Ed25519 half gives false."""
    import oracle
    from circl_b200.eddsa import EdDilithium2
    s = EdDilithium2()
    dpk, dsk = oracle.mldsa_keygen(2, bytes(range(32)))
    dsig = [oracle.mldsa_sign(2, dsk, c[2])[0] for c in cases]
    pks = _rows([dpk + c[1] for c in cases])
    ok = s.VerifyBatch(pks, [c[2] for c in cases], _rows([d + c[3] for d, c in zip(dsig, cases)]))
    assert not _names_of_mismatches(cases, ok)
    good = [i for i, c in enumerate(cases) if c[4]]
    bad = []
    for j, i in enumerate(good):
        d = bytearray(dsig[i])
        d[(37 * j) % 2420] ^= 1 << (j % 8)
        assert not oracle.mldsa_verify(2, dpk, cases[i][2], bytes(d))
        bad.append(bytes(d) + cases[i][3])
    assert not s.VerifyBatch(pks[good], [cases[i][2] for i in good], _rows(bad)).any()
