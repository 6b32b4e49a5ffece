"""Host model of the ML-KEM matrix sampler's staging (csrc/mlkem.cu: uniform_block, sample_kernel, sample_fix_kernel)
and the search for SHAKE128 streams at its edges, shared by tests/test_mlkem_sampler_staging_model.py (CPU) and
tests/test_gpu_mlkem_sampler_staging.py.

The model follows the kernel index for index: the warp's flat staging (lane l's 120 int16 entries from 120 l), the
carried partial chunk, the packed per-stream job word of the write passes and the half-warp to stream mapping, the
clamp from the third block on, and the hand-off of a short stream to the fix kernel.  Staging and output start out
as garbage, so a chunk that is never written, or written from the wrong entries, shows up as a wrong coefficient."""
import hashlib

import numpy as np

Q = 3329
N = 256
CAND = 112  # 12-bit candidates per 168-byte block
STAGE = 120  # int16 entries of staging per thread (kStageChunks = 15 chunks of 8)


def candidates(seed: bytes, x: int, y: int, blocks: int) -> np.ndarray:
    """(blocks, 112) candidates of XOF(seed || x || y), in the order sample.go parses them."""
    b = np.frombuffer(hashlib.shake_128(seed + bytes([x, y])).digest(168 * blocks), dtype=np.uint8).astype(np.int32)
    g = b.reshape(-1, 3)
    d1 = g[:, 0] | ((g[:, 1] & 0xF) << 8)
    d2 = (g[:, 1] >> 4) | (g[:, 2] << 4)
    return np.stack([d1, d2], axis=1).reshape(blocks, CAND)


def completion(seed: bytes, x: int, y: int) -> int:
    """1-based index of the candidate that brings the stream to 256 coefficients (336 = last of block 3)."""
    c = candidates(seed, x, y, 6).reshape(-1)
    return int(np.searchsorted(np.cumsum(c < Q), N) + 1)


# the edges of the staging: a fourth block; 256 on the last candidate of block 3; 256 within the first 80 of block 3
KINDS = {
    "four_blocks": lambda done: done > 3 * CAND,
    "exact_block3_end": lambda done: done == 3 * CAND,
    "early_block3": lambda done: 2 * CAND < done <= 2 * CAND + 80,
}


def find_rho(kind: str, tag: bytes, k: int, count: int, skip: int = 0):
    """`count` seeded 32-byte seeds, each with at least one matrix stream (x, y < k) of the kind; returns
    [(rho, [(x, y), ...])].  The search is deterministic in (kind, tag, k)."""
    want = KINDS[kind]
    out, i = [], 0
    while len(out) < count + skip:
        rho = hashlib.shake_256(tag + kind.encode() + i.to_bytes(4, "little")).digest(32)
        hits = [(x, y) for x in range(k) for y in range(k) if want(completion(rho, x, y))]
        if hits:
            out.append((rho, hits))
        i += 1
    return out[skip:]


def _warp_blocks(lanes_cand, live, poly, stage, out, fixed):
    """Run uniform_block over one warp.  lanes_cand: (32, B, 112); poly: (32,) polynomial index of each lane in `out`
    (flat int16, 256 per polynomial).  Returns the per-lane counts."""
    lanes = np.arange(32)
    cnt = np.zeros(32, dtype=np.int64)
    b = 0
    while True:
        checked = b >= 2
        base = cnt & ~7
        wp = cnt - base
        end = N - base
        for f in range(CAND):
            d = lanes_cand[:, b, f]
            if checked:
                idx = np.minimum(wp, end)
            else:
                assert (wp < end).all()  # the unclamped blocks never reach coefficient 256
                idx = wp
            assert (idx < STAGE).all()
            stage[lanes * STAGE + idx] = d
            wp = wp + (d < Q)
        cnt = base + np.minimum(wp, end)
        nch = (cnt - base + 7) >> 3
        assert (nch <= 15).all()
        job = np.where(live, ((32 * poly + base // 8) << 4) | nch, 0)
        assert (job < 2**32).all()
        for q in range(16):  # pass q: lanes 0-15 write stream 2q, lanes 16-31 stream 2q + 1
            half, c = lanes >> 4, lanes & 15
            jp = job[2 * q + half]
            on = c < (jp & 15)
            src = (half * 15 + c + 2 * q * 15)[on]  # chunk of the warp's staging (rd[2 q kStageChunks])
            dst = ((jp >> 4) + c)[on]
            out.reshape(-1, 8)[dst] = stage.reshape(-1, 8)[src]
        keep = cnt < N
        for ln in lanes[keep]:  # the partial last chunk to the front
            k8 = ((cnt[ln] - base[ln]) >> 3) * 8
            stage[ln * STAGE:ln * STAGE + 8] = stage[ln * STAGE + k8:ln * STAGE + k8 + 8].copy()
        b += 1
        if (fixed and b == 3) or (not fixed and not (cnt < N).any()):
            return cnt


def _fix(cands, got, row):
    """sample_fix_kernel: squeeze on from block 4 and append from position `got`."""
    cnt = int(got)
    for d in cands[3:].reshape(-1):
        if cnt == N:
            break
        if d < Q:
            row[cnt] = d
            cnt += 1
    assert cnt == N


def sample_matrix(rhos, k: int, transpose: bool, seed: int = 0) -> np.ndarray:
    """launch_sample over nkeys = len(rhos) keys: sample_kernel (3 blocks per warp, 128-thread CTAs, one thread per
    stream s = (i k + j) nkeys + key, dead lanes and warps as in the kernel) and sample_fix_kernel.  Returns
    A[key][i][j] as (nkeys, k, k, 256) int16."""
    rng = np.random.default_rng(seed)
    nkeys = len(rhos)
    total = nkeys * k * k
    out = rng.integers(-(1 << 15), 1 << 15, size=nkeys * k * k * N).astype(np.int64)
    stage = rng.integers(-(1 << 15), 1 << 15, size=32 * STAGE).astype(np.int64)
    cache = {}

    def cand(key, ij):
        i, j = divmod(ij, k)
        x, y = (i, j) if transpose else (j, i)
        if (key, ij) not in cache:
            cache[(key, ij)] = candidates(rhos[key], x, y, 6)
        return cache[(key, ij)]

    for w0 in range(0, total, 32):  # warps; a CTA is 4 of them and shares nothing between them
        s = w0 + np.arange(32)
        live = s < total
        sc = np.where(live, s, total - 1)
        key, ij = sc % nkeys, sc // nkeys
        lc = np.stack([cand(int(a), int(b)) for a, b in zip(key, ij)])
        poly = key * k * k + ij
        got = _warp_blocks(lc, live, poly, stage, out, True)
        for ln in np.nonzero(live & (got < N))[0]:
            p = int(poly[ln])
            _fix(lc[ln], got[ln], out[p * N:(p + 1) * N])
    return out.reshape(nkeys, k, k, N).astype(np.int16)


def derive_uniform(seeds, xy, seed: int = 0) -> np.ndarray:
    """derive_uniform_kernel: every warp runs blocks until its streams are all full; polynomials relative to the
    warp's first.  Returns (n, 256) int16."""
    rng = np.random.default_rng(seed)
    n = len(seeds)
    out = rng.integers(-(1 << 15), 1 << 15, size=n * N).astype(np.int64)
    stage = rng.integers(-(1 << 15), 1 << 15, size=32 * STAGE).astype(np.int64)
    for w0 in range(0, n, 32):
        s = w0 + np.arange(32)
        live = s < n
        sc = np.where(live, s, n - 1)
        lc = np.stack([candidates(seeds[i], int(xy[i][0]), int(xy[i][1]), 8) for i in sc])
        wout = out[w0 * N:]  # a view: the kernel's `out` is polys + (s - lane) * N
        _warp_blocks(lc, live, sc - w0, stage, wout, False)
    return out.reshape(n, N).astype(np.int16)
