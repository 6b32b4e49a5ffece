"""FrodoKEM-640-SHAKE on the GPU against the oracle (oracle/frodo.c) and the reference's PQCgenKAT transcript hash:
per-op keys, one key shared by the batch (the tensor-core path), implicit rejection, private keys whose S holds
arbitrary 16-bit values, numpy and CUDA-tensor inputs."""
import numpy as np
import pytest

import frodo_model as M
from conftest import load_golden

pytestmark = pytest.mark.gpu

PK, SK, CT, SS = 9616, 19888, 9720, 16


@pytest.fixture(scope="module")
def kem():
    import circl_b200
    from circl_b200 import frodo
    circl_b200.init(0)
    yield frodo.Scheme()


@pytest.fixture(scope="module")
def O():
    from oracle import frodo as oracle_frodo
    return oracle_frodo


def _spots(n):
    return sorted({0, n // 3, n // 2, n - 1})


def test_pqcgenkat_transcript_on_gpu(kem):
    want = load_golden("frodo_vectors.json.gz")["kats"][0]
    rows = lambda xs: np.stack([np.frombuffer(x, np.uint8) for x in xs])  # noqa: E731
    def keygen(ks):
        pk, sk = kem.DeriveKeyPairBatch(rows(ks))
        return [r.tobytes() for r in pk], [r.tobytes() for r in sk]
    def encaps(pks, es):
        ct, ss = kem.EncapsulateBatch(rows(pks), rows(es))
        return [r.tobytes() for r in ct], [r.tobytes() for r in ss]
    def decaps(sks, cts):
        return [r.tobytes() for r in kem.DecapsulateBatch(rows(sks), rows(cts))]
    assert M.kat_hash(keygen, encaps, decaps, name=want["name"]) == want["sha256"]


@pytest.mark.parametrize("n", [1, 33, 1500])
def test_parity_per_op_keys(kem, O, n):
    rng = np.random.default_rng(n)
    seeds = rng.integers(0, 256, size=(n, 48), dtype=np.uint8)
    pk, sk = kem.DeriveKeyPairBatch(seeds)
    es = rng.integers(0, 256, size=(n, 16), dtype=np.uint8)
    ct, ss = kem.EncapsulateBatch(pk, es)
    for i in _spots(n):
        assert (pk[i].tobytes(), sk[i].tobytes()) == O.keygen(seeds[i].tobytes()), i
        assert (ct[i].tobytes(), ss[i].tobytes()) == O.encaps(pk[i].tobytes(), es[i].tobytes()), i
    assert np.array_equal(kem.DecapsulateBatch(sk, ct), ss)
    # implicit rejection: a flipped bit in the B' part and in the C part of every other ciphertext
    bad = ct.copy()
    idx = np.arange(0, n, 2)
    bad[idx, rng.integers(0, 9600)] ^= 1
    if n > 1:
        bad[idx[1::2], 9600 + rng.integers(0, 120)] ^= 0x80
    got = kem.DecapsulateBatch(sk, bad)
    for i in _spots(n) + [int(idx[-1])]:
        assert got[i].tobytes() == O.decaps(sk[i].tobytes(), bad[i].tobytes()), i
    assert not np.array_equal(got[idx], ss[idx])
    assert np.array_equal(got[1::2], ss[1::2])


def test_arbitrary_keys(kem, O):
    """S with any 16-bit value, and a public key made of arbitrary bytes: no validation, as in the reference."""
    rng = np.random.default_rng(7)
    n = 40
    sk = rng.integers(0, 256, size=(n, SK), dtype=np.uint8)
    pk = rng.integers(0, 256, size=(n, PK), dtype=np.uint8)
    ct = rng.integers(0, 256, size=(n, CT), dtype=np.uint8)
    es = rng.integers(0, 256, size=(n, 16), dtype=np.uint8)
    ss = kem.DecapsulateBatch(sk, ct)
    gct, gss = kem.EncapsulateBatch(pk, es)
    for i in (0, 17, n - 1):
        assert ss[i].tobytes() == O.decaps(sk[i].tobytes(), ct[i].tobytes()), i
        assert (gct[i].tobytes(), gss[i].tobytes()) == O.encaps(pk[i].tobytes(), es[i].tobytes()), i
    # a valid key pair whose S is replaced by arbitrary values still decapsulates like the oracle
    kp, ks = kem.DeriveKeyPairBatch(rng.integers(0, 256, size=(n, 48), dtype=np.uint8))
    kct, _ = kem.EncapsulateBatch(kp, es)
    ks[:, 16 + PK:16 + PK + 10240] = rng.integers(0, 256, size=(n, 10240), dtype=np.uint8)
    got = kem.DecapsulateBatch(ks, kct)
    for i in (0, 5, n - 1):
        assert got[i].tobytes() == O.decaps(ks[i].tobytes(), kct[i].tobytes()), i


def test_cuda_tensors(kem, O):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(3)
    n = 33
    seeds = rng.integers(0, 256, size=(n, 48), dtype=np.uint8)
    es = rng.integers(0, 256, size=(n, 16), dtype=np.uint8)
    hpk, hsk = kem.DeriveKeyPairBatch(seeds)
    hct, hss = kem.EncapsulateBatch(hpk, es)
    dpk, dsk = kem.DeriveKeyPairBatch(torch.from_numpy(seeds).cuda())
    dct, dss = kem.EncapsulateBatch(dpk, torch.from_numpy(es).cuda())
    dss2 = kem.DecapsulateBatch(dsk, dct)
    torch.cuda.synchronize()
    assert np.array_equal(dpk.cpu().numpy(), hpk) and np.array_equal(dsk.cpu().numpy(), hsk)
    assert np.array_equal(dct.cpu().numpy(), hct) and np.array_equal(dss.cpu().numpy(), hss)
    assert np.array_equal(dss2.cpu().numpy(), hss)
    # one shared key on the device path
    pk0, sk0 = kem.UnmarshalBinaryPublicKey(hpk[0].tobytes()), kem.UnmarshalBinaryPrivateKey(hsk[0].tobytes())
    sct, sss = kem.EncapsulateBatch(pk0, torch.from_numpy(es).cuda())
    back = kem.DecapsulateBatch(sk0, sct)
    torch.cuda.synchronize()
    assert (sct[n - 1].cpu().numpy().tobytes(), sss[n - 1].cpu().numpy().tobytes()) == O.encaps(hpk[0].tobytes(),
                                                                                                 es[n - 1].tobytes())
    assert torch.equal(back, sss)


def test_shared_key_path_equals_full_stride(kem, O):
    """Stride 0 (A once per call, S'A as one GEMM) gives the same bytes as the key repeated at full stride."""
    rng = np.random.default_rng(12)
    n = 1 << 12
    pk, sk = kem.DeriveKeyPairBatch(rng.integers(0, 256, size=(1, 48), dtype=np.uint8))
    es = rng.integers(0, 256, size=(n, 16), dtype=np.uint8)
    pko, sko = kem.UnmarshalBinaryPublicKey(pk[0].tobytes()), kem.UnmarshalBinaryPrivateKey(sk[0].tobytes())
    ct0, ss0 = kem.EncapsulateBatch(pko, es)
    ct1, ss1 = kem.EncapsulateBatch(np.repeat(pk, n, axis=0), es)
    assert np.array_equal(ct0, ct1) and np.array_equal(ss0, ss1)
    for i in _spots(n):
        assert (ct0[i].tobytes(), ss0[i].tobytes()) == O.encaps(pk[0].tobytes(), es[i].tobytes()), i
    bad = ct0.copy()
    bad[::3, rng.integers(0, 9600, size=1)] ^= 4       # B' part
    bad[1::3, 9600 + rng.integers(0, 120, size=1)] ^= 2  # C part
    d0 = kem.DecapsulateBatch(sko, bad)
    d1 = kem.DecapsulateBatch(np.repeat(sk, n, axis=0), bad)
    assert np.array_equal(d0, d1)
    assert np.array_equal(d0[2::3], ss0[2::3]) and not np.any(np.all(d0[::3] == ss0[::3], axis=1))
    for i in (0, 1, n - 1):
        assert d0[i].tobytes() == O.decaps(sk[0].tobytes(), bad[i].tobytes()), i


def test_sub_batches_past_the_chunk(kem, O):
    """n = 8193 crosses the 8192-op sub-batch of device-pointer calls (seed, key, ct and ss offsets of the second
    sub-batch; the shared key's H(pk) kept in work row 0) and the 4096-op staging chunk of host-pointer calls: spot
    checks against the oracle at 8191, 8192 and n - 1, and host results equal to device results."""
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(8193)
    n = 8193
    seeds = rng.integers(0, 256, size=(n, 48), dtype=np.uint8)
    es = rng.integers(0, 256, size=(n, 16), dtype=np.uint8)
    spots = [0, 4095, 4096, 8191, 8192]
    dpk, dsk = kem.DeriveKeyPairBatch(torch.from_numpy(seeds).cuda())
    dct, dss = kem.EncapsulateBatch(dpk, torch.from_numpy(es).cuda())
    bad = dct.clone()
    bad[8192::2, 100] ^= 1
    dss2 = kem.DecapsulateBatch(dsk, bad)
    pk0, sk0 = kem.UnmarshalBinaryPublicKey(dpk[5].cpu().numpy().tobytes()), \
        kem.UnmarshalBinaryPrivateKey(dsk[5].cpu().numpy().tobytes())
    sct, sss = kem.EncapsulateBatch(pk0, torch.from_numpy(es).cuda())
    sbad = sct.clone()
    sbad[8191:, 9650] ^= 2
    sss2 = kem.DecapsulateBatch(sk0, sbad)
    torch.cuda.synchronize()
    pk, sk, ct, ss = (x.cpu().numpy() for x in (dpk, dsk, dct, dss))
    scth, sssh, bad_h, sbad_h = sct.cpu().numpy(), sss.cpu().numpy(), bad.cpu().numpy(), sbad.cpu().numpy()
    d2, sd2 = dss2.cpu().numpy(), sss2.cpu().numpy()
    for i in spots:
        assert (pk[i].tobytes(), sk[i].tobytes()) == O.keygen(seeds[i].tobytes()), i
        assert (ct[i].tobytes(), ss[i].tobytes()) == O.encaps(pk[i].tobytes(), es[i].tobytes()), i
        assert d2[i].tobytes() == O.decaps(sk[i].tobytes(), bad_h[i].tobytes()), i
        assert (scth[i].tobytes(), sssh[i].tobytes()) == O.encaps(pk[5].tobytes(), es[i].tobytes()), i
        assert sd2[i].tobytes() == O.decaps(sk[5].tobytes(), sbad_h[i].tobytes()), i
    assert np.array_equal(d2[:8192], ss[:8192]) and np.array_equal(d2[8193:], ss[8193:])
    assert not np.array_equal(d2[8192], ss[8192])
    assert np.array_equal(sd2[:8191], sssh[:8191]) and not np.any(np.all(sd2[8191:] == sssh[8191:], axis=1))
    # the same operations from host arrays (staged in chunks of 4096)
    hpk, hsk = kem.DeriveKeyPairBatch(seeds)
    assert np.array_equal(hpk, pk) and np.array_equal(hsk, sk)
    hct, hss = kem.EncapsulateBatch(hpk, es)
    assert np.array_equal(hct, ct) and np.array_equal(hss, ss)
    assert np.array_equal(kem.DecapsulateBatch(hsk, bad_h), d2)
    h2ct, h2ss = kem.EncapsulateBatch(pk0, es)
    assert np.array_equal(h2ct, scth) and np.array_equal(h2ss, sssh)
    assert np.array_equal(kem.DecapsulateBatch(sk0, sbad_h), sd2)
