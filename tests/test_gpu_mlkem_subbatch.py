"""GPU parity across the sub-batch boundaries of the ML-KEM flows: KeyGen, Encapsulate (per-op keys, one of them not
canonical) and Decapsulate (one dk whose ek part is not canonical, with a matching H(ek)) over 2 kSub + 37 ops, every
op against the oracle.  The K-PKE kernels sample their noise themselves from the seed of their op, so an off-by-one
in the per-sub-batch seed offsets shows up here as wrong ciphertexts after the first sub-batch."""
import hashlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

KSUB = 8192  # kSub of circl_b200/csrc/mlkem.cu
N = 2 * KSUB + 37
KS = {"ML-KEM-512": 2, "ML-KEM-768": 3, "ML-KEM-1024": 4}


@pytest.fixture(scope="module")
def cb():
    import circl_b200
    circl_b200.init(0)
    yield circl_b200
    circl_b200.shutdown()


def _bytes(tag, n, width):
    return np.frombuffer(hashlib.shake_256(tag).digest(n * width), dtype=np.uint8).reshape(n, width)


@pytest.mark.parametrize("ps", list(KS))
def test_keygen_encaps_decaps_across_sub_batches(cb, ps):
    import oracle
    from circl_b200 import mlkem
    k = KS[ps]
    scheme = mlkem.ByName(ps)
    seeds = _bytes(b"subbatch-keygen" + ps.encode(), N, 64)
    ek, dk = scheme.DeriveKeyPairBatch(seeds)
    for i in range(N):
        wek, wdk = oracle.mlkem_keygen(k, seeds[i].tobytes())
        assert ek[i].tobytes() == wek and dk[i].tobytes() == wdk, i

    # Encapsulate: op `bad` (last of the first sub-batch) gets a first coefficient of 4095 >= q -> kem.ErrPubKey,
    # a zero ciphertext and shared secret for that op, the others unaffected
    bad = KSUB - 1
    eks = ek.copy()
    eks[bad, 0], eks[bad, 1] = 0xFF, eks[bad, 1] | 0x0F
    ms = _bytes(b"subbatch-m" + ps.encode(), N, 32)
    ct = np.empty((N, scheme.CiphertextSize()), dtype=np.uint8)
    ss = np.empty((N, 32), dtype=np.uint8)
    with pytest.raises(mlkem.ErrPubKey) as ei:
        scheme.EncapsulateBatch(eks, ms, ct=ct, ss=ss)
    want = np.zeros(N, dtype=np.uint8)
    want[bad] = 1
    assert np.array_equal(ei.value.status, want)
    wct, wss, fails = oracle.mlkem_encaps_batch(k, eks, ms, nthreads=8)
    assert fails == 1
    ok = np.arange(N) != bad
    assert np.array_equal(ct[ok], wct[ok]) and np.array_equal(ss[ok], wss[ok])
    assert not ct[bad].any() and not ss[bad].any()

    # Decapsulate: every third ciphertext corrupted (implicit rejection); dk of op `bad2` (first of the last, partial
    # sub-batch) carries the non-canonical ek with its own H(ek), which the re-encryption parses leniently
    bad2 = 2 * KSUB
    dks = dk.copy()
    ekoff = 384 * k
    eklen = 384 * k + 32
    dks[bad2, ekoff], dks[bad2, ekoff + 1] = 0xFF, dks[bad2, ekoff + 1] | 0x0F
    dks[bad2, ekoff + eklen:ekoff + eklen + 32] = np.frombuffer(
        hashlib.sha3_256(dks[bad2, ekoff:ekoff + eklen].tobytes()).digest(), dtype=np.uint8)
    cts = wct.copy()
    cts[::3, 7] ^= 0x20
    got = scheme.DecapsulateBatch(dks, cts)
    for i in range(N):
        assert got[i].tobytes() == oracle.mlkem_decaps(k, dks[i].tobytes(), cts[i].tobytes()), i
