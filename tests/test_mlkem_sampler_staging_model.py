"""The index arithmetic of the ML-KEM matrix sampler's per-block staging (csrc/mlkem.cu uniform_block), run as a host
model (tests/mlkem_uniform_model.py) against the oracle's DeriveUniform: sample_kernel + sample_fix_kernel for
KeyGen's A and Encapsulate's A^T, with a partial last CTA, a single key and seeds rigged to the edges of the staging
(a fourth block, 256 on the last candidate of block 3, 256 early in block 3) at lanes 0 and 31 of their warps; and
derive_uniform_kernel, which runs every stream to the end itself."""
import numpy as np
import pytest

import mlkem_uniform_model as model

K = 3


@pytest.fixture(scope="module")
def orc():
    import oracle
    oracle.build()
    return oracle


def _rigged(k, count):
    return {kind: model.find_rho(kind, b"staging-model", k, count) for kind in model.KINDS}


def _check_matrix(orc, rhos, k, transpose):
    A = model.sample_matrix(rhos, k, transpose, seed=len(rhos))
    for key, rho in enumerate(rhos):
        for i in range(k):
            for j in range(k):
                x, y = (i, j) if transpose else (j, i)
                assert np.array_equal(A[key, i, j], orc.kyber_derive_uniform(rho, x, y)), (key, i, j)


@pytest.mark.parametrize("transpose", [True, False])
def test_sample_kernel_model_with_rigged_keys(orc, transpose):
    rng = np.random.default_rng(203)
    nkeys = 256  # 2304 streams, 18 CTAs; stream (ij, key) sits at lane key % 32
    rhos = [rng.bytes(32) for _ in range(nkeys)]
    rig = _rigged(K, 2)
    places = {"four_blocks": (0, 127), "exact_block3_end": (31, 128), "early_block3": (96, 255)}
    for kind, (p0, p1) in places.items():
        rhos[p0], rhos[p1] = rig[kind][0][0], rig[kind][1][0]
    _check_matrix(orc, rhos, K, transpose)


@pytest.mark.parametrize("k", [2, 3, 4])
def test_sample_kernel_model_partial_cta_and_single_key(orc, k):
    rng = np.random.default_rng(k)
    rig = _rigged(k, 1)
    rhos = [rng.bytes(32) for _ in range(37)]  # 37 k^2 streams: a partial last CTA, dead lanes and warps
    rhos[36] = rig["four_blocks"][0][0]
    rhos[0] = rig["exact_block3_end"][0][0]
    _check_matrix(orc, rhos, k, True)
    _check_matrix(orc, [rig["four_blocks"][0][0]], k, True)  # one key: k^2 live threads
    _check_matrix(orc, [rig["exact_block3_end"][0][0]], k, False)


def test_derive_uniform_model(orc):
    rng = np.random.default_rng(236)
    n = 300  # the last warp has 12 live lanes
    seeds = [rng.bytes(32) for _ in range(n)]
    xy = rng.integers(0, 4, size=(n, 2)).tolist()
    rig = _rigged(K, 2)
    for pos, kind, r in ((0, "four_blocks", 0), (31, "four_blocks", 1), (127, "exact_block3_end", 0),
                         (128, "early_block3", 0), (299, "four_blocks", 0)):
        rho, hits = rig[kind][r]
        seeds[pos], xy[pos] = rho, list(hits[0])
    got = model.derive_uniform(seeds, xy, seed=1)
    for i in range(n):
        assert np.array_equal(got[i], orc.kyber_derive_uniform(seeds[i], xy[i][0], xy[i][1])), i
