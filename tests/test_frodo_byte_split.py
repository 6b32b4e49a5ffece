"""CPU check of the identity behind frodo_gemm_kernel (circl_b200/csrc/frodo.cu): with A = lo + 256 hi its two byte
planes (u8) and S' sampled in [-12, 12] (s8),

    S' A = S' lo + 256 (S' hi)   (mod 2^16),

where each int32 sum of the tensor cores is exact because |sum| <= 640 * 255 * 12 < 2^21.  Checked on the extreme
operands (A = 0xFFFF, S' = +-12) and on random ones against a direct product mod 2^16."""
import numpy as np

N = 640


def _split_product(sp, a):
    lo, hi = a & 0xFF, a >> 8
    p_lo, p_hi = sp @ lo, sp @ hi
    for p in (p_lo, p_hi):
        assert np.abs(p).max() < 2 ** 21                  # exact in int32
        assert np.abs(p).max() <= N * 255 * 12
    return (p_lo + (p_hi << 8)) & 0xFFFF


def test_extreme_operands():
    a = np.full((N, N), 0xFFFF, dtype=np.int64)
    for s in (12, -12):
        sp = np.full((8, N), s, dtype=np.int64)
        got = _split_product(sp, a)
        assert np.array_equal(got, (sp @ a) & 0xFFFF)
        assert np.abs(sp @ (a & 0xFF)).max() == N * 255 * 12
    sp = np.where(np.arange(N) % 2 == 0, 12, -12)[None, :].repeat(8, 0).astype(np.int64)
    assert np.array_equal(_split_product(sp, a), (sp @ a) & 0xFFFF)


def test_random_operands():
    rng = np.random.default_rng(4)
    for _ in range(4):
        a = rng.integers(0, 65536, size=(N, N), dtype=np.int64)
        sp = rng.integers(-12, 13, size=(64, N), dtype=np.int64)
        want = np.zeros((64, N), dtype=np.uint16)
        for j in range(N):  # the reference's uint16 accumulation, row by row of A
            want = (want + (sp[:, j:j + 1].astype(np.uint16) * a[j].astype(np.uint16))).astype(np.uint16)
        assert np.array_equal(_split_product(sp, a), want.astype(np.int64))
