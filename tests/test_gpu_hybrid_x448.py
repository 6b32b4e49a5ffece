"""GPU parity for Kyber768-X448 and Kyber1024-X448 (kem/hybrid/hybrid.go:83-93 over xkem.go) against the oracle,
shaped like test_gpu_hybrid.test_hybrid_vs_oracle_and_low_order_points, plus device pointers with the 8-byte-aligned
rows these layouts have and host-pointer sharding over two GPUs."""
import hashlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

NAMES = ["Kyber768-X448", "Kyber1024-X448"]
LOW = (1).to_bytes(56, "little")  # a point of order 4 on the twist (curve.go:76-104)


@pytest.fixture(scope="module")
def cb():
    import circl_b200
    circl_b200.init(0)
    yield circl_b200
    circl_b200.shutdown()


def _rows(items):
    return np.frombuffer(b"".join(items), dtype=np.uint8).reshape(len(items), -1)


def _h(tag, i, n):
    return hashlib.shake_256(bytes([tag]) + i.to_bytes(8, "little")).digest(n)


@pytest.mark.parametrize("name", NAMES)
def test_hybrid_x448_vs_oracle_and_low_order_points(cb, name):
    from oracle import x448 as ox
    from circl_b200 import mlkem, x448
    s = x448.ByName(name)
    assert s.Name() == name
    assert (s.PublicKeySize(), s.PrivateKeySize(), s.CiphertextSize()) == ox.hybrid_sizes(name)
    assert (s.SharedKeySize(), s.EncapsulationSeedSize(), s.SeedSize()) == ox.hybrid_seed_sizes(name) + (64,)
    n = 400
    seeds = _rows([_h(5, i, 64) for i in range(n)])
    eseeds = _rows([_h(6, i, 56) for i in range(n)])
    pk, sk = s.DeriveKeyPairBatch(seeds)
    ct, ss = s.EncapsulateBatch(pk, eseeds)
    assert ss.shape == (n, 88)
    assert (s.DecapsulateBatch(sk, ct) == ss).all()
    for i in list(range(0, n, 37)) + [n - 1]:
        assert (pk[i].tobytes(), sk[i].tobytes()) == ox.hybrid_keygen(name, seeds[i].tobytes())
        assert (ct[i].tobytes(), ss[i].tobytes(), 0) == ox.hybrid_encaps(name, pk[i].tobytes(), eseeds[i].tobytes())
    # single calls with key objects; a shared-key batch
    p0, s0 = s.DeriveKeyPair(seeds[0].tobytes())
    c0, k0 = s.EncapsulateDeterministically(p0, eseeds[0].tobytes())
    assert (c0, k0) == (ct[0].tobytes(), ss[0].tobytes()) and s.Decapsulate(s0, c0) == k0
    cs, ks = s.EncapsulateBatch(p0, eseeds[:33])
    assert (s.DecapsulateBatch(s0, cs) == ks).all()
    assert cs[5].tobytes() == ox.hybrid_encaps(name, p0.MarshalBinary(), eseeds[5].tobytes())[0]
    # implicit rejection: a flipped byte in the Kyber half changes only the Kyber half of the secret
    bad = ct[:16].copy()
    bad[:, 300] ^= 1
    ss_bad = s.DecapsulateBatch(sk[:16], bad)
    assert (ss_bad[:, :56] == ss[:16, :56]).all() and (ss_bad[:, 56:] != ss[:16, 56:]).any(axis=1).all()
    assert ss_bad[3].tobytes() == ox.hybrid_decaps(name, sk[3].tobytes(), bad[3].tobytes())[0]
    # a low-order X448 share is kem.ErrPubKey on both sides, per op
    bad_pk = pk[:8].copy()
    bad_pk[3, :56] = np.frombuffer(LOW, dtype=np.uint8)
    with pytest.raises(mlkem.ErrPubKey) as ei:
        s.EncapsulateBatch(bad_pk, eseeds[:8])
    assert ei.value.status.tolist() == [0, 0, 0, 1, 0, 0, 0, 0]
    bad_ct = ct[:8].copy()
    bad_ct[5, :56] = 0
    with pytest.raises(mlkem.ErrPubKey) as ei:
        s.DecapsulateBatch(sk[:8], bad_ct)
    assert (ei.value.status != 0).tolist() == [False] * 5 + [True] + [False] * 2
    assert ox.hybrid_decaps(name, sk[5].tobytes(), bad_ct[5].tobytes())[1] == 1


@pytest.mark.parametrize("name", NAMES)
def test_device_pointers_8_byte_aligned_rows(cb, name):
    import torch
    from oracle import x448 as ox
    from circl_b200 import x448
    s = x448.ByName(name)
    n = 3000
    g = torch.Generator(device="cpu").manual_seed(12)
    seeds = torch.randint(0, 256, (n, 64), dtype=torch.uint8, generator=g).cuda()
    eseeds = torch.randint(0, 256, (n, 56), dtype=torch.uint8, generator=g).cuda()
    pk, sk = s.DeriveKeyPairBatch(seeds)
    ct, ss = s.EncapsulateBatch(pk, eseeds)
    ss2 = s.DecapsulateBatch(sk, ct)
    torch.cuda.synchronize()
    assert [t.stride(0) % 16 for t in (pk, sk, ct)] == [8, 8, 8]  # rows 8- but not 16-byte aligned
    assert torch.equal(ss, ss2)
    for i in (0, 1777, n - 1):
        sd, es = seeds[i].cpu().numpy().tobytes(), eseeds[i].cpu().numpy().tobytes()
        opk, osk = ox.hybrid_keygen(name, sd)
        assert (pk[i].cpu().numpy().tobytes(), sk[i].cpu().numpy().tobytes()) == (opk, osk)
        assert (ct[i].cpu().numpy().tobytes(), ss[i].cpu().numpy().tobytes(), 0) == ox.hybrid_encaps(name, opk, es)


def test_host_pointers_shard_over_two_gpus():
    import circl_b200
    from circl_b200 import _ffi, x448
    if _ffi.lib().cb200_device_count() < 2:
        pytest.skip("needs two GPUs")
    from oracle import x448 as ox
    circl_b200.shutdown()
    circl_b200.init_devices(2)
    try:
        s = x448.ByName("Kyber768-X448")
        n = 40000  # above two shards of the host pipeline's minimum
        seeds = np.frombuffer(hashlib.shake_256(b"shard").digest(64 * n), dtype=np.uint8).reshape(n, 64)
        eseeds = np.frombuffer(hashlib.shake_256(b"eshard").digest(56 * n), dtype=np.uint8).reshape(n, 56)
        pk, sk = s.DeriveKeyPairBatch(seeds)
        ct, ss = s.EncapsulateBatch(pk, eseeds)
        assert (s.DecapsulateBatch(sk, ct) == ss).all()
        for i in (0, n // 2 + 3, n - 1):
            assert (ct[i].tobytes(), ss[i].tobytes(), 0) == ox.hybrid_encaps("Kyber768-X448", pk[i].tobytes(),
                                                                                 eseeds[i].tobytes())
    finally:
        circl_b200.shutdown()
