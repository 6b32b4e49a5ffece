"""GPU parity at the edges of the ML-KEM matrix sampler's per-block staging (csrc/mlkem.cu uniform_block): keys whose
rho makes a matrix stream need a fourth SHAKE128 block (finished by sample_fix_kernel), reach 256 coefficients on the
last candidate of block 3, or reach 256 early in block 3 -- found on the host with hashlib (tests/mlkem_uniform_model.py)
and built into canonical keys as a real key's t-hat || the chosen rho -- placed at lanes 0 and 31 of their warps, at the
first and last thread of a CTA and on both sides of the sub-batch boundaries.  Encapsulate with per-op keys and with one
shared key, derive_uniform on the same streams, and KeyGen -> Encapsulate -> Decapsulate (A, not A^T, and the
re-encryption) across a sub-batch boundary, every output against the oracle."""
import hashlib

import numpy as np
import pytest

import mlkem_uniform_model as model

pytestmark = pytest.mark.gpu

KSUB = 8192  # kSub of circl_b200/csrc/mlkem.cu
KS = {"ML-KEM-512": 2, "ML-KEM-768": 3, "ML-KEM-1024": 4}
# ops whose streams sit at lane 0 / lane 31 of a warp; 127 / 128 are the last / first thread of a CTA, 8191 / 8192 and
# 16383 / 16384 the last / first op of a sub-batch (the last sub-batch, of 37 ops, numbers its streams differently)
PLACES = [0, 31, 32, 63, 96, 127, 128, 159, 8160, 8191, 8192, 8223, 16352, 16383, 16384, 16385, 16419, 16420]
KINDS = list(model.KINDS)


@pytest.fixture(scope="module")
def cb():
    import circl_b200
    circl_b200.init(0)
    yield circl_b200
    circl_b200.shutdown()


def _bytes(tag, n, width):
    return np.frombuffer(hashlib.shake_256(tag).digest(n * width), dtype=np.uint8).reshape(n, width)


def _rigged(k):
    """kind -> [(rho, hits)], enough for every place the kind takes"""
    return {kind: model.find_rho(kind, b"staging-gpu", k, len(PLACES) // len(KINDS)) for kind in KINDS}


def _keys(k, n, tag):
    """n canonical eks: the t-hat of four real keys, each op with its own seeded rho"""
    import oracle
    t = [oracle.mlkem_keygen(k, hashlib.shake_256(tag + bytes([i])).digest(64))[0][:384 * k] for i in range(4)]
    rho = _bytes(tag + b"rho", n, 32)
    return np.stack([np.frombuffer(t[i % 4] + rho[i].tobytes(), dtype=np.uint8) for i in range(n)])


@pytest.mark.parametrize("ps", list(KS))
def test_encaps_per_op_keys_with_rigged_streams(cb, ps):
    import oracle
    from circl_b200 import mlkem
    k = KS[ps]
    n = 2 * KSUB + 37
    scheme = mlkem.ByName(ps)
    eks = _keys(k, n, b"staging-ek" + ps.encode())
    rig = _rigged(k)
    rigged = []
    for i, op in enumerate(PLACES):  # every kind lands at lane 0 and at lane 31
        rho, _ = rig[KINDS[i % 3]][i // 3]
        eks[op, 384 * k:] = np.frombuffer(rho, dtype=np.uint8)
        rigged.append(op)
    ms = _bytes(b"staging-m" + ps.encode(), n, 32)
    ct, ss = scheme.EncapsulateBatch(eks, ms)
    wct, wss, fails = oracle.mlkem_encaps_batch(k, eks, ms, nthreads=8)
    assert fails == 0
    for op in rigged:
        assert ct[op].tobytes() == wct[op].tobytes() and ss[op].tobytes() == wss[op].tobytes(), op
    bad = np.nonzero((ct != wct).any(axis=1) | (ss != wss).any(axis=1))[0]
    assert bad.size == 0, bad[:10]


@pytest.mark.parametrize("ps", list(KS))
def test_encaps_shared_key_with_rigged_streams(cb, ps):
    import oracle
    from circl_b200 import mlkem
    k = KS[ps]
    scheme = mlkem.ByName(ps)
    t = _keys(k, 1, b"staging-shared" + ps.encode())[0, :384 * k].tobytes()
    ms = _bytes(b"staging-shared-m" + ps.encode(), 300, 32)
    for kind, found in _rigged(k).items():
        ek = t + found[0][0]
        ct, ss = scheme.EncapsulateBatch(scheme.UnmarshalBinaryPublicKey(ek), ms)
        wct, wss, fails = oracle.mlkem_encaps_batch(k, np.frombuffer(ek, dtype=np.uint8), ms, nthreads=4)
        assert fails == 0 and np.array_equal(ct, wct) and np.array_equal(ss, wss), kind


def test_derive_uniform_with_rigged_streams(cb):
    import oracle
    from circl_b200 import kyber
    rng = np.random.default_rng(236)
    n = 300  # the last warp has 12 live lanes
    seeds = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
    xy = rng.integers(0, 4, size=(n, 2), dtype=np.uint8)
    rig = _rigged(3)
    for i, pos in enumerate([0, 31, 32, 63, 127, 128, 255, 256, 287, 288, 298, 299]):
        rho, hits = rig[KINDS[i % 3]][i // 3 % len(rig[KINDS[i % 3]])]
        seeds[pos] = np.frombuffer(rho, dtype=np.uint8)
        xy[pos] = hits[-1]
    got = kyber.derive_uniform(seeds, xy)
    for i in range(n):
        assert np.array_equal(got[i], oracle.kyber_derive_uniform(seeds[i].tobytes(), int(xy[i, 0]), int(xy[i, 1]))), i


def test_keygen_encaps_decaps_across_a_sub_batch(cb):
    # KeyGen's rho comes out of G(d) and cannot be chosen: seeded random d, about 1 % of the streams are short
    import oracle
    from circl_b200 import mlkem
    n = KSUB + 301
    scheme = mlkem.ByName("ML-KEM-768")
    seeds = _bytes(b"staging-keygen", n, 64)
    ek, dk = scheme.DeriveKeyPairBatch(seeds)
    short = 0
    for i in range(n):
        wek, wdk = oracle.mlkem_keygen(3, seeds[i].tobytes())
        assert ek[i].tobytes() == wek and dk[i].tobytes() == wdk, i
        if i % 64 == 0:
            rho = wek[-32:]
            short += sum(model.completion(rho, x, y) > 3 * model.CAND for x in range(3) for y in range(3))
    assert short > 0  # the sample above did include streams that sample_fix_kernel finished
    ms = _bytes(b"staging-keygen-m", n, 32)
    ct, ss = scheme.EncapsulateBatch(ek, ms)
    wct, wss, fails = oracle.mlkem_encaps_batch(3, ek, ms, nthreads=8)
    assert fails == 0 and np.array_equal(ct, wct) and np.array_equal(ss, wss)
    cts = ct.copy()
    cts[1::5, 3] ^= 0x01  # implicit rejection on every fifth op: the re-encryption must differ from ct
    got = scheme.DecapsulateBatch(dk, cts)
    ok = np.ones(n, dtype=bool)
    ok[1::5] = False
    assert np.array_equal(got[ok], ss[ok])
    for i in range(0, n, 37):
        assert got[i].tobytes() == oracle.mlkem_decaps(3, dk[i].tobytes(), cts[i].tobytes()), i
    for i in range(1, n, 5 * 31):
        assert got[i].tobytes() == oracle.mlkem_decaps(3, dk[i].tobytes(), cts[i].tobytes()), i
