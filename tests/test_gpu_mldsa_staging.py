"""GPU parity of ML-DSA Sign / Verify / KeyGen where the batch is cut and staged, against the oracle (byte-exact).

- The host-pointer sign path stages chunks of 2^16 signatures through three rotating slots (messages rebased per chunk,
  the next chunk's inputs in flight while the current one runs its rejection loop); verify stages chunks of 2^15 and
  keygen chunks of 2^14.  The batches here cross those boundaries.
- Device pointers through the C ABI: padded and shared key rows, rnd, context strings, Sign_internal, status bytes and
  the attempt count, each byte-equal to the host path on the same inputs, and the argument errors of that path.
- mu = SHAKE256(tr || 0 || len(ctx) || ctx || M) with the end of its input just before, at and just after a boundary of
  the 136-byte rate, on the host and the device path.
"""
import concurrent.futures as cf
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

INTERNAL = 1           # CB200_SIGN_INTERNAL
ERR_ARG = -1           # CB200_ERR_ARG
SIZES = {44: (1312, 2560, 2420), 65: (1952, 4032, 3309), 87: (2592, 4896, 4627), 3: (1952, 4000, 3293)}
NAMES = {44: "ML-DSA-44", 65: "ML-DSA-65", 87: "ML-DSA-87", 3: "Dilithium3"}


@pytest.fixture(scope="module")
def cb():
    import circl_b200
    circl_b200.init(0)
    yield circl_b200
    circl_b200.shutdown()


def _pmap(fn, *cols):
    """fn over rows, in threads (the oracle's ctypes calls release the GIL)."""
    with cf.ThreadPoolExecutor(16) as ex:
        return list(ex.map(fn, *cols))


def _bytes(rng, n, width):
    return rng.integers(0, 256, size=(n, width), dtype=np.uint8)


def _msgs(lens, seed):
    """Messages of the given lengths, cut from one seeded random blob."""
    lens = np.asarray(lens, dtype=np.int64)
    blob = np.random.default_rng(seed).integers(0, 256, size=int(lens.sum()), dtype=np.uint8).tobytes()
    off = np.concatenate([[0], np.cumsum(lens)])
    return [blob[off[i]:off[i + 1]] for i in range(len(lens))]


def _pool(mode, count, seed):
    from circl_b200 import mldsa
    return mldsa.ByName(NAMES[mode]).DeriveKeyBatch(_bytes(np.random.default_rng(seed), count, 32))


# ---------------------------------------------------------------- the C ABI on host arrays or on CUDA copies of them
def _blob(msgs):
    off = np.zeros(len(msgs) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(m) for m in msgs])
    return np.frombuffer(b"".join(msgs) + bytes(8), dtype=np.uint8), off   # 8 bytes of read padding


class _Side:
    """Buffers of one call, either the numpy arrays themselves or device copies of them."""

    def __init__(self, device):
        self.device, self.keep = device, []

    def __call__(self, a):
        if a is None:
            return None
        if not self.device:
            a = np.ascontiguousarray(a)
            self.keep.append(a)
            return a.ctypes.data
        import torch
        t = torch.from_numpy(np.array(a, dtype=a.dtype, order="C").view(np.uint8)).cuda()   # a writable copy
        self.keep.append(t)
        return t.data_ptr()

    def out(self, ptr_index, shape, dtype=np.uint8):
        """The i-th buffer handed out, read back as a numpy array."""
        b = self.keep[ptr_index]
        if self.device:
            import torch
            torch.cuda.synchronize()
            b = b.cpu().numpy()
        return b.view(dtype).reshape(shape).copy()

    def begin(self):
        if self.device:
            import torch
            from circl_b200 import _ffi
            _ffi.check(_ffi.lib().cb200_set_stream(torch.cuda.current_stream().cuda_stream))


def _ctx_arg(ctx):
    buf = (C.c_uint8 * max(1, len(ctx))).from_buffer_copy(ctx or b"\0")
    return buf, (C.cast(buf, C.c_void_p) if ctx else None)


def _sign(mode, sk, stride, msgs, ctx=b"", rnd=None, flags=0, device=False):
    """cb200_mldsa_sign -> (sig, status, attempts).  The outputs start out as 0xCC / 0xEE so unwritten bytes show."""
    from circl_b200 import _ffi
    n, sigsz = len(msgs), SIZES[mode][2]
    s = _Side(device)
    s.begin()
    blob, off = _blob(msgs)
    p = [s(sk), s(blob), s(off), s(rnd), s(np.full((n, sigsz), 0xCC, np.uint8)), s(np.full(n, 0xEE, np.uint8))]
    att = C.c_uint64(0)
    cbuf, cptr = _ctx_arg(ctx)
    _ffi.check(_ffi.lib().cb200_mldsa_sign(mode, p[0], stride, p[1], p[2], cptr, len(ctx), p[3], p[4], p[5], n, flags,
                                           C.cast(C.pointer(att), C.c_void_p)))
    iout = 4 if rnd is not None else 3   # index of sig among the buffers kept (rnd may be absent)
    return s.out(iout, (n, sigsz)), s.out(iout + 1, (n,)), int(att.value)


def _verify(mode, pk, stride, msgs, sig, ctx=b"", flags=0, device=False):
    from circl_b200 import _ffi
    n = len(msgs)
    s = _Side(device)
    s.begin()
    blob, off = _blob(msgs)
    p = [s(pk), s(blob), s(off), s(sig), s(np.full(n, 0xEE, np.uint8))]
    cbuf, cptr = _ctx_arg(ctx)
    _ffi.check(_ffi.lib().cb200_mldsa_verify(mode, p[0], stride, p[1], p[2], cptr, len(ctx), p[3], p[4], n, flags))
    ok = s.out(4, (n,))
    assert set(np.unique(ok).tolist()) <= {0, 1}
    return ok.astype(bool)


def _keygen(mode, seeds, device=False):
    from circl_b200 import _ffi
    n, (pksz, sksz, _) = len(seeds), SIZES[mode]
    s = _Side(device)
    s.begin()
    p = [s(seeds), s(np.full((n, pksz), 0xCC, np.uint8)), s(np.full((n, sksz), 0xCC, np.uint8))]
    _ffi.check(_ffi.lib().cb200_mldsa_keygen(mode, p[0], p[1], p[2], n))
    return s.out(1, (n, pksz)), s.out(2, (n, sksz))


def _oracle_sign(mode, sk, msg, ctx=b"", rnd=None, internal=False):
    import oracle
    return oracle.mldsa_sign(mode, bytes(sk), msg, ctx=ctx, rnd=bytes(32) if rnd is None else bytes(rnd),
                             internal=internal)[0]


# ---------------------------------------------------------------- 1. sign across the 2^16 chunk, per-op keys
def test_sign_across_one_chunk_boundary_per_op_keys(cb):
    import oracle
    from circl_b200 import mldsa
    scheme = mldsa.ByName("ML-DSA-65")
    n = (1 << 16) + 3
    _, pool = _pool(65, 64, 11)
    idx = np.arange(n) % 64
    lens = (np.arange(n) * 131) % 701                                  # 0 .. 700 bytes
    edge = [65535, 65536, n - 1]                                       # last of chunk 0, first and last of chunk 1
    assert len({int(idx[i]) for i in edge}) == 3 and len({int(lens[i]) for i in edge}) == 3
    sks = pool[idx]
    msgs = _msgs(lens, 12)
    rnd = _bytes(np.random.default_rng(13), n, 32)
    sig, attempts = scheme.SignBatch(sks, msgs, rnd=rnd, return_attempts=True)
    want, want_attempts = oracle.mldsa_sign_batch(65, sks, msgs, rnd, nthreads=16)
    bad = np.flatnonzero((sig != want).any(axis=1))
    assert bad.size == 0, f"{bad.size} signatures differ, first rows {bad[:8].tolist()}"
    assert attempts == want_attempts
    print(f"\nsign 2^16 + 3, per-op keys: {attempts} attempts ({attempts / n:.3f} per signature)")


# ---------------------------------------------------------------- 2. sign across four chunks, one shared key
def test_sign_across_four_chunks_shared_key(cb):
    import oracle
    from circl_b200 import mldsa
    scheme = mldsa.ByName("ML-DSA-65")
    K = 1 << 16
    n = 4 * K + 1                                 # chunks 0..3 full (chunk 3 reuses slot 0), chunk 4 a single op
    i = np.arange(n)
    lens = np.empty(n, dtype=np.int64)
    lens[:K] = (i[:K] * 53) % 211                 # mixed
    lens[K:2 * K] = 0                             # all empty: no message bytes to stage for the chunk
    lens[2 * K:3 * K] = i[2 * K:3 * K] % 29       # short ...
    long_row = 2 * K + 4321
    lens[long_row] = 9000                         # ... but one long message sizes the staging area
    lens[3 * K:4 * K] = (i[3 * K:4 * K] * 97) % 389
    lens[n - 1] = 77
    msgs = _msgs(lens, 21)
    pk, sk = scheme.DeriveKey(bytes(range(32)))
    rnd = _bytes(np.random.default_rng(22), n, 32)   # with one key and empty messages only rnd tells the ops apart
    sig, attempts = scheme.SignBatch(sk, msgs, rnd=rnd, return_attempts=True)
    assert 3.5 < attempts / n < 7.0
    rows = sorted({0, K - 1, K, 2 * K, long_row, 3 * K - 1, 3 * K, n - 1} | set(range(0, n, 997)))
    want = _pmap(lambda r: _oracle_sign(65, sk.MarshalBinary(), msgs[r], rnd=rnd[r]), rows)
    bad = [r for r, w in zip(rows, want) if sig[r].tobytes() != w]
    assert not bad, f"rows differing from the oracle: {bad[:8]}"
    assert scheme.VerifyBatch(pk, msgs, sig).all()
    # distinct c~ for every op (hence distinct signatures): the empty-message chunk 1 relies on rnd alone, and a chunk
    # that read another chunk's rnd or message bytes would repeat that chunk's signatures
    ct = np.ascontiguousarray(sig[:, :48]).view(np.uint64)
    assert np.unique(ct, axis=0).shape[0] == n
    print(f"\nsign 4 * 2^16 + 1, shared key: {attempts} attempts ({attempts / n:.3f} per signature)")


# ---------------------------------------------------------------- 3. verify (chunks of 2^15) and keygen (2^14)
def test_verify_across_its_chunk_boundary(cb):
    import oracle
    from circl_b200 import mldsa
    scheme = mldsa.ByName("ML-DSA-65")
    n = (1 << 15) + 2
    ctx = b"staging"
    pool_pk, pool_sk = _pool(65, 64, 31)
    idx = np.arange(n) % 64
    pks = pool_pk[idx]
    msgs = _msgs((np.arange(n) * 41) % 300, 32)
    sig = scheme.SignBatch(pool_sk[idx], msgs, ctx=ctx)
    sig[(1 << 15) - 1, 5] ^= 0x01                 # c~ of the last op of chunk 0
    sig[1 << 15, 0] ^= 0x80                       # c~ of the first op of chunk 1
    sig[n - 1] = np.frombuffer(_oracle_sign(65, pool_sk[idx[n - 1]], msgs[n - 1], ctx=ctx + b"!"), dtype=np.uint8)
    ok = scheme.VerifyBatch(pks, msgs, sig, ctx=ctx)
    want = _pmap(lambda r: oracle.mldsa_verify(65, pks[r].tobytes(), msgs[r], sig[r].tobytes(), ctx=ctx), range(n))
    assert ok.tolist() == want
    assert np.flatnonzero(~ok).tolist() == [(1 << 15) - 1, 1 << 15, n - 1]


def test_keygen_across_its_chunk_boundary(cb):
    import oracle
    from circl_b200 import mldsa
    n = (1 << 14) + 1
    seeds = _bytes(np.random.default_rng(41), n, 32)
    pk, sk = mldsa.ByName("ML-DSA-65").DeriveKeyBatch(seeds)
    rows = sorted({(1 << 14) - 1, 1 << 14} | set(range(0, n, 331)))
    want = _pmap(lambda r: oracle.mldsa_keygen(65, seeds[r].tobytes()), rows)
    assert [(pk[r].tobytes(), sk[r].tobytes()) for r in rows] == want


# ---------------------------------------------------------------- 4. device pointers through the C ABI
def _padded(rows, fill=0xA5):
    """rows in a buffer of stride (row size rounded up to 16) + 16, the pad bytes set to `fill`."""
    width = rows.shape[1]
    stride = (width + 15) // 16 * 16 + 16
    out = np.full((rows.shape[0], stride), fill, dtype=np.uint8)
    out[:, :width] = rows
    return out, stride


@pytest.mark.parametrize("mode", [44, 65, 87, 3])
def test_device_pointers_match_the_host_path(cb, mode):
    import oracle
    nist = mode > 10
    pksz, sksz, _ = SIZES[mode]
    n = 40
    rng = np.random.default_rng(50 + mode)
    seeds = _bytes(rng, n, 32)
    pk, sk = _keygen(mode, seeds)
    pk_d, sk_d = _keygen(mode, seeds, device=True)
    assert np.array_equal(pk_d, pk) and np.array_equal(sk_d, sk)
    for r in (0, 17, n - 1):
        assert (pk[r].tobytes(), sk[r].tobytes()) == oracle.mldsa_keygen(mode, seeds[r].tobytes())

    msgs = _msgs((np.arange(n) * 37) % 300, 51 + mode)
    rnd = _bytes(rng, n, 32)
    ctx = bytes((7 * j + 1) & 0xFF for j in range(255)) if nist else b""
    skp, stride = _padded(sk)
    configs = [  # (keys, stride, key of op i, rnd, ctx, flags)
        (skp, stride, lambda i: sk[i], rnd, ctx, 0),                                  # padded rows, rnd, 255-byte ctx
        (sk[5], 0, lambda i: sk[5], None, b"", INTERNAL if nist else 0),             # shared key, Sign_internal
        (sk, sksz, lambda i: sk[i], rnd, b"\x01" if nist else b"", 0),                # packed rows, 1-byte ctx
    ]
    sigs = []
    for keys, kstride, key, r, c, flags in configs:
        sig_h, st_h, att_h = _sign(mode, keys, kstride, msgs, ctx=c, rnd=r, flags=flags)
        sig_d, st_d, att_d = _sign(mode, keys, kstride, msgs, ctx=c, rnd=r, flags=flags, device=True)
        assert np.array_equal(sig_d, sig_h)
        assert not st_h.any() and not st_d.any()
        assert att_d == att_h and att_h >= n
        rows = list(range(0, n, 7)) + [n - 1]
        want = _pmap(lambda i: _oracle_sign(mode, key(i), msgs[i], ctx=c, rnd=None if r is None else r[i],
                                            internal=bool(flags)), rows)
        assert [sig_h[i].tobytes() for i in rows] == want
        sigs.append(sig_h)

    # verify: padded pk rows and per-op signatures of config 0, three of them tampered
    pkp, pstride = _padded(pk)
    bad = sigs[0].copy()
    bad[3, 0] ^= 1
    bad[11, 200] ^= 0x10
    bad[n - 1, -1] ^= 1
    ok_h = _verify(mode, pkp, pstride, msgs, bad, ctx=ctx)
    ok_d = _verify(mode, pkp, pstride, msgs, bad, ctx=ctx, device=True)
    want = _pmap(lambda i: oracle.mldsa_verify(mode, pk[i].tobytes(), msgs[i], bad[i].tobytes(), ctx=ctx), range(n))
    assert ok_h.tolist() == want and ok_d.tolist() == want
    assert not want[3] and not want[11] and sum(want) >= n - 3
    # verify: shared pk, the Sign_internal signatures of config 1, one of them on a changed message
    flags = INTERNAL if nist else 0
    m2 = list(msgs)
    m2[9] = m2[9][:-1] + bytes([m2[9][-1] ^ 1])
    ok_h = _verify(mode, pk[5], 0, m2, sigs[1], flags=flags)
    ok_d = _verify(mode, pk[5], 0, m2, sigs[1], flags=flags, device=True)
    assert ok_h.tolist() == ok_d.tolist() == [i != 9 for i in range(n)]
    assert not oracle.mldsa_verify(mode, pk[5].tobytes(), m2[9], sigs[1][9].tobytes(), internal=bool(flags))


def test_device_argument_errors(cb):
    """Argument errors of the device-pointer path: returned before anything is launched."""
    import torch
    from circl_b200 import _ffi
    L = _ffi.lib()
    _ffi.check(L.cb200_set_stream(torch.cuda.current_stream().cuda_stream))
    pksz, sksz, sigsz = SIZES[65]
    n = 4
    sk = torch.zeros((n, sksz + 16), dtype=torch.uint8, device="cuda")
    pk = torch.zeros((n, pksz + 16), dtype=torch.uint8, device="cuda")
    blob = torch.zeros(64, dtype=torch.uint8, device="cuda")
    off = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    sig = torch.zeros((n, sigsz), dtype=torch.uint8, device="cuda")
    ok = torch.zeros(n, dtype=torch.uint8, device="cuda")
    off_h = np.zeros(n + 1, dtype=np.uint64)
    blob_h = np.zeros(64, dtype=np.uint8)
    launches = cb.launch_count()

    def err(rc, text):
        assert rc == ERR_ARG
        assert text in L.cb200_last_error().decode()

    # device keys and signatures with host messages
    err(L.cb200_mldsa_sign(65, sk.data_ptr(), sksz, blob_h.ctypes.data, off_h.ctypes.data, None, 0, None,
                           sig.data_ptr(), None, n, 0, None), "mixed host/device pointers")
    err(L.cb200_mldsa_verify(65, pk.data_ptr(), pksz, blob.data_ptr(), off_h.ctypes.data, None, 0, sig.data_ptr(),
                             ok.data_ptr(), n, 0), "mixed host/device pointers")
    # 2^24 signatures on device buffers of four rows: the count is refused before any row is touched
    err(L.cb200_mldsa_sign(65, sk.data_ptr(), 0, blob.data_ptr(), off.data_ptr(), None, 0, None, sig.data_ptr(), None,
                           1 << 24, 0, None), "limited to 2^24 - 1 signatures")
    # key strides that are not a multiple of 16
    err(L.cb200_mldsa_sign(65, sk.data_ptr(), sksz + 8, blob.data_ptr(), off.data_ptr(), None, 0, None,
                           sig.data_ptr(), None, n, 0, None), "16-byte aligned")
    err(L.cb200_mldsa_verify(65, pk.data_ptr(), pksz + 8, blob.data_ptr(), off.data_ptr(), None, 0, sig.data_ptr(),
                             ok.data_ptr(), n, 0), "16-byte aligned")
    assert cb.launch_count() == launches
    torch.cuda.synchronize()
    assert not sig.any().item() and not ok.any().item()


# ---------------------------------------------------------------- 5. mu at the SHAKE256 rate edges
RATE = 136


def _edge_messages(prefix):
    """(k, mlen): the absorbed prefix + mlen bytes end one byte before, at and one byte after the k-th rate boundary."""
    return [(k, RATE * k + d - prefix) for k in (1, 2, 3, 5) for d in (-1, 0, 1) if RATE * k + d - prefix >= 0]


@pytest.mark.parametrize("mode", [65, 87, 3])
def test_mu_at_the_rate_edges(cb, mode):
    import oracle
    nist = mode > 10
    pk, sk = _pool(mode, 1, 60 + mode)
    pk, sk = pk[0], sk[0]
    trlen = 64 if nist else 32
    variants = ([(c, False) for c in (b"", b"\x2a", bytes(range(255)))] + [(b"", True)]) if nist else [(b"", False)]
    for ctx, internal in variants:
        prefix = trlen + (2 + len(ctx) if nist and not internal else 0)
        edges = _edge_messages(prefix)
        n = len(edges)
        assert n >= 6
        msgs = _msgs([m for _, m in edges], 61 + len(ctx) + internal)
        assert all(((prefix + len(m)) % RATE) in (RATE - 1, 0, 1) for m in msgs)
        rnd = _bytes(np.random.default_rng(62 + len(ctx)), n, 32)
        flags = INTERNAL if internal else 0
        want = _pmap(lambda i: _oracle_sign(mode, sk, msgs[i], ctx=ctx, rnd=rnd[i], internal=internal), range(n))
        for device in (False, True):
            sig, status, _ = _sign(mode, sk, 0, msgs, ctx=ctx, rnd=rnd, flags=flags, device=device)
            assert [s.tobytes() for s in sig] == want, (ctx, internal, device)
            assert not status.any()
            assert _verify(mode, pk, 0, msgs, sig, ctx=ctx, flags=flags, device=device).all()
            # one byte changed next to the boundary (the message's last byte when it ends before it)
            bent = []
            for (k, mlen), m in zip(edges, msgs):
                j = min(mlen - 1, RATE * k - 1 - prefix)
                bent.append(m[:j] + bytes([m[j] ^ 0x40]) + m[j + 1:])
            assert not _verify(mode, pk, 0, bent, sig, ctx=ctx, flags=flags, device=device).any()
        assert not oracle.mldsa_verify(mode, pk.tobytes(), bent[0], bytes(want[0]), ctx=ctx, internal=internal)
