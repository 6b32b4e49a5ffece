"""The OPRF servers across their host staging chunks, on one GPU, with every output row checked against
tests/oprf_model.py.

Layout: row i of a batch uses input combination i mod P (a small prime).  A combination fixes the key, r, the element
tuple and the input, so the model computes P combinations and every row has a known answer; a row staged at a shifted
offset, a wrong key stride or a mixed-up slot changes values.  P divides no chunk of any schedule used here (asserted).
The first and the last row of every staging chunk is an invalid op (an element that does not decode, sk = 0 or n,
r = 0, t = 0 in mode 2), which must fail only itself with the model's status bits and all-zero outputs.

Covered: Evaluate with the ramp engaged (m = 8), an odd chunk (m = 3), m = 1, many elements per request (past 256,
where the composite index I2OSP(j, 2) needs both bytes) and one request per chunk (m = 16385); DeriveKeyBatch over
the ramp with info of 0, 1 and 65535 bytes; FullEvaluate over every input length from 0 to 306 and at 65534 and 65535
bytes; info at its limit in every entry point and refused past it; per-op keys in wider rows (sk_stride > Ns).  Every
batch also runs on CUDA tensors, whose results must equal the host results byte for byte.
"""
import random

import numpy as np
import pytest

import oprf_model as om

gpu = pytest.mark.gpu  # every test but the schedule mirror runs on the GPU

IDENT = ["P256-SHA256", "P384-SHA384", "P521-SHA512"]
P = 31                 # input combinations per batch
CB200_ERR_ARG = -1     # include/circl_b200.h
INFO_MAX = bytes(range(256)) * 255 + bytes(range(255))  # 65535 bytes, the largest info (I2OSP(len(info), 2))


# ---------------------------------------------------------------- the staging schedule on one GPU
def eval_chunk(m):
    """Requests per staged Evaluate chunk (oprf.cu evaluate: max(1, 2^15 / m))."""
    return max(1, (1 << 15) // m)


OP_CHUNK = 1 << 15  # DeriveKey and FullEvaluate ops per staged chunk (oprf.cu derive and full)


def staged(n, chunk):
    """(first, count) of every chunk of a host batch through run_staged (api.cu): once n >= 6 chunk and
    chunk >= 4096, chunks of chunk/4, chunk/4, chunk/2 lead and their mirror image trails the full chunks."""
    ramp = [chunk // 4, chunk // 4, chunk // 2] if n >= 6 * chunk and chunk >= 4096 else []
    left = n - 2 * sum(ramp)
    counts = ramp + [min(chunk, left - f) for f in range(0, left, chunk)] + ramp[::-1]
    return list(zip(np.cumsum([0] + counts[:-1]).tolist(), counts))


def msg_chunks(n, chunk=OP_CHUNK):
    """(first, count) of every chunk of a host batch with messages: run_msgs (flow_internal.h), no ramp."""
    return [(f, min(chunk, n - f)) for f in range(0, n, chunk)]


def edges(sched, period=P):
    """The first and the last row of every chunk; asserts that the period divides no chunk."""
    assert all(c % period for _, c in sched if c > 1), (period, sched)
    return sorted({f for f, _ in sched} | {f + c - 1 for f, c in sched})


def test_schedule_mirror():
    s = staged(6 * 4096 + 37, 4096)
    assert [c for _, c in s] == [1024, 1024, 2048, 4096, 4096, 4096, 4096, 37, 2048, 1024, 1024]
    assert sum(c for _, c in s) == 6 * 4096 + 37 and s[-1][0] + s[-1][1] == 6 * 4096 + 37
    assert [c for _, c in staged(3 * 10922 + 5, 10922)] == [10922, 10922, 10922, 5]  # 10922 < 6 chunk: no ramp
    assert [c for _, c in staged(5, eval_chunk(16385))] == [1, 1, 1, 1, 1]  # one request per chunk
    assert eval_chunk(1 << 16) == 1 and eval_chunk(300) == 109


# ---------------------------------------------------------------- inputs and the model
@pytest.fixture(scope="module")
def cb():
    import circl_b200
    circl_b200.init(0)  # one GPU: for_each_shard makes one shard, so the schedule above is the whole batch's
    yield circl_b200
    circl_b200.shutdown()


@pytest.fixture(params=IDENT, ids=["p256", "p384", "p521"])
def suite(request, cb):
    from circl_b200 import oprf
    return om.SUITES[request.param], oprf.GetSuite(request.param)


def _sc(rng, s):
    return om.i2osp(rng.randrange(1, s.n), s.Ns)


def _rows(blist, width=None):
    a = np.frombuffer(b"".join(blist), dtype=np.uint8)
    return a.reshape(len(blist), -1 if width is None else width).copy()


def _bad_elements(s):
    """Encodings that do not decode: a bad prefix, X = p, and an X with no point."""
    x = next(v for v in range(1, 200) if not om._is_square(s, (v ** 3 - 3 * v + s.b) % s.p))
    return [b"\x04" + om.i2osp(s.g[0], s.nbytes), b"\x02" + om.i2osp(s.p, s.nbytes), b"\x03" + om.i2osp(x, s.nbytes)]


def _same(got, want, what):
    got = np.asarray(got)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = np.nonzero((got != want).reshape(want.shape[0], -1).any(axis=1))[0]
    assert bad.size == 0, f"{what}: {bad.size} of {want.shape[0]} rows differ, first {bad[:8].tolist()}"


def _np(t):
    return t.cpu().numpy() if hasattr(t, "cpu") else t


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


class EvalBatch:
    """n requests of m elements in the layout above, with the model's expected evaluations, proofs and status
    bytes.  per_op: one key per request (else one key for the batch); bad_rows get an invalid op each."""

    def __init__(self, s, mode, m, n, per_op, info, seed, bad_rows):
        rng = random.Random(seed)
        Ne = s.Ne
        pool = [om.compress(s, om.mul(s, rng.randrange(1, s.n), s.g)) for _ in range(3)]
        tup = np.random.default_rng(seed).integers(0, len(pool), size=(P, m))
        ktab = [_sc(rng, s) for _ in range(P if per_op else 1)]
        rtab = [_sc(rng, s) for _ in range(P)]
        btab = np.frombuffer(b"".join(pool), dtype=np.uint8).reshape(len(pool), Ne)[tup].reshape(P, m * Ne)
        evtab = np.zeros((P, m * Ne), np.uint8)
        prtab = np.zeros((P, 2 * s.Ns), np.uint8)
        idx = np.arange(n) % P
        for c in sorted(set(idx.tolist())):  # only the combinations a short batch uses
            ev, pr = om.evaluate_grouped(s, mode, ktab[c if per_op else 0], [pool[j] for j in tup[c]],
                                         rtab[c] if mode else None, info)
            evtab[c] = np.frombuffer(b"".join(ev), np.uint8)
            if mode:
                prtab[c] = np.frombuffer(pr, np.uint8)
        self.K = _rows(ktab)[idx] if per_op else _rows(ktab).reshape(-1)
        self.B, self.R = btab[idx], _rows(rtab)[idx]
        self.EV, self.PR, self.ST = evtab[idx], prtab[idx], np.zeros(n, np.uint8)
        kinds = ["element"] + (["sk0", "skn"] if per_op else []) + (["r0"] if mode else []) + \
            (["t0"] if mode == om.PARTIAL and per_op else [])
        bad = _bad_elements(s)
        for q, i in enumerate(bad_rows):
            kind = kinds[q % len(kinds)]
            if kind == "element":  # at a varying position, the last one included
                j = (m - 1) if q % 2 else (q * 7919) % m
                self.B[i, j * Ne:(j + 1) * Ne] = np.frombuffer(bad[q % 3], np.uint8)
            elif kind == "r0":
                self.R[i] = 0
            else:
                k = {"sk0": 0, "skn": s.n, "t0": s.n - om.info_scalar(s, info)}[kind]
                self.K[i] = np.frombuffer(om.i2osp(k, s.Ns), np.uint8)
            sk = self.K[i].tobytes() if per_op else self.K.tobytes()
            els = [self.B[i, j * Ne:(j + 1) * Ne].tobytes() for j in range(m)]
            with pytest.raises(om.OprfError) as e:
                om.evaluate_grouped(s, mode, sk, els, self.R[i].tobytes() if mode else None, info)
            self.ST[i], self.EV[i], self.PR[i] = e.value.status, 0, 0
        self.s, self.mode, self.m, self.info = s, mode, m, info

    def run(self, S, dev):
        """(evaluated, proof, status) as numpy arrays, through EvaluateBatch on host arrays or CUDA tensors."""
        from circl_b200 import oprf
        args = [_cuda(a) if dev else a for a in (self.K, self.B, self.R)]
        try:
            ev, pr = oprf.EvaluateBatch(S, self.mode, args[0], args[1], self.m, args[2] if self.mode else None,
                                        self.info)
            st = np.zeros(len(self.ST), np.uint8)
        except oprf.OprfError as e:
            (ev, pr), st = e.results, _np(e.status)
        return _np(ev), (_np(pr) if self.mode else None), st

    def check(self, got, what):
        ev, pr, st = got
        _same(st, self.ST, what + " status")
        _same(ev, self.EV, what + " evaluations")
        if self.mode:
            _same(pr, self.PR, what + " proofs")


def _host_and_device(S, b):
    host = b.run(S, False)
    b.check(host, "host")
    dev = b.run(S, True)
    for h, d in zip(host, dev):
        if h is not None:
            assert np.array_equal(h, d)  # the device call (one launch over all n) equals the staged one


# ---------------------------------------------------------------- Evaluate
@gpu
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_evaluate_ramp_and_slot_wrap(suite, mode):
    """m = 8: chunks of 4096 requests; 6 * 4096 + 37 engages the ramp and takes every slot several times.  Per-op
    keys; mode 2 with the largest info."""
    s, S = suite
    m, n = 8, 6 * 4096 + 37
    b = EvalBatch(s, mode, m, n, True, INFO_MAX if mode == 2 else b"", 100 + mode, edges(staged(n, eval_chunk(m))))
    _host_and_device(S, b)


@gpu
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_evaluate_odd_chunk_shared_key(suite, mode):
    """m = 3: chunks of 10922 = 2 * 43 * 127 requests, one shared key."""
    s, S = suite
    m, n = 3, 3 * 10922 + 5
    b = EvalBatch(s, mode, m, n, False, b"odd chunk" if mode == 2 else b"", 200 + mode,
                  edges(staged(n, eval_chunk(m))))
    _host_and_device(S, b)


@gpu
@pytest.mark.parametrize("mode", [1, 2])
def test_evaluate_one_element_per_request(suite, mode):
    """m = 1: chunks of 2^15 requests, 2^16 + 3 of them with per-op keys."""
    s, S = suite
    m, n = 1, (1 << 16) + 3
    b = EvalBatch(s, mode, m, n, True, b"m = 1" if mode == 2 else b"", 300 + mode, edges(staged(n, eval_chunk(m))))
    _host_and_device(S, b)


# Many elements per request in modes 1 and 2: m past 256, where I2OSP(j, 2) in the composite weights uses its high
# byte, and n over three chunks of 2^15 / 300 = 109 requests.  The composite kernel loops over a request's m elements
# in one thread, so a call's time grows with m: at m = 300 a P-521 call takes about 10 s on an H100, and m = 16385 (one
# request per chunk) would take minutes.  That chunk size is tested in mode 0, which has no composite.
MANY_M, MANY_N = 300, 2 * 109 + 3


@gpu
@pytest.mark.parametrize("mode", [1, 2])
def test_evaluate_many_elements_per_request(suite, mode):
    s, S = suite
    m, n = MANY_M, MANY_N
    sched = staged(n, eval_chunk(m))
    assert len(sched) >= 3
    b = EvalBatch(s, mode, m, n, True, b"many" if mode == 2 else b"", 400 + mode, edges(sched))
    assert b.ST.any() and not b.ST.all()
    _host_and_device(S, b)


@gpu
def test_evaluate_one_request_per_chunk(suite):
    """Mode 0 at m = 16385: max(1, 2^15 / m) = 1, so every request is a chunk of its own and the three slots rotate
    one request at a time; each element is one thread of oprf_eval_kernel.  Every row is the first and the last of
    its chunk, so only rows 1 and 3 of the 5 get an invalid op."""
    s, S = suite
    m, n = 16385, 5
    sched = staged(n, eval_chunk(m))
    assert [c for _, c in sched] == [1] * n
    b = EvalBatch(s, 0, m, n, True, b"", 450, edges(sched)[1::2])
    assert [i for i in range(n) if b.ST[i]] == [1, 3]
    _host_and_device(S, b)


# ---------------------------------------------------------------- DeriveKeyBatch
@gpu
@pytest.mark.parametrize("mode,info", [(0, b""), (1, b"\x00"), (2, INFO_MAX)], ids=["info0", "info1", "info65535"])
def test_derive_key_batch_ramp(suite, mode, info):
    """6 * 2^15 + 11 seeds (the ramp engaged) tiled from a table of P, sk and pk checked on every row."""
    from circl_b200 import oprf
    s, S = suite
    n = 6 * OP_CHUNK + 11
    edges(staged(n, OP_CHUNK))
    rng = random.Random(500 + mode)
    seeds = [bytes(rng.randrange(256) for _ in range(32)) for _ in range(P)]
    want = [om.derive_key(s, mode, x, info) for x in seeds]
    idx = np.arange(n) % P
    SEEDS, SK, PK = _rows(seeds)[idx], _rows([w[0] for w in want])[idx], _rows([w[1] for w in want])[idx]
    sk, pk = oprf.DeriveKeyBatch(S, mode, SEEDS, info)
    _same(sk, SK, "host sk")
    _same(pk, PK, "host pk")
    dsk, dpk = oprf.DeriveKeyBatch(S, mode, _cuda(SEEDS), info)
    _same(_np(dsk), SK, "device sk")
    _same(_np(dpk), PK, "device pk")


# ---------------------------------------------------------------- FullEvaluate
# FullEvaluate combinations: one per input length 0..306.  Those 307 consecutive lengths take every residue mod 64 and
# mod 128, so the Finalize hash and expand_message_xmd's b_0, which hold the input after a fixed prefix, meet every
# block and length-padding edge of SHA-256 (64-byte blocks) and SHA-384/512 (128-byte blocks).
Q = 307


def _inputs_table():
    rng = random.Random(600)
    return [bytes(rng.randrange(256) for _ in range(n)) for n in range(Q)]


@gpu
@pytest.mark.parametrize("per_op", [True, False], ids=["per_op", "shared"])
@pytest.mark.parametrize("mode", [0, 2])
def test_full_evaluate_across_chunks(suite, mode, per_op):
    """2 * 2^15 + 77 ops, every input length from 0 to 306; inputs of 65535 and 65534 bytes and invalid keys at the
    chunk edges; the largest info (mode 0 must ignore it)."""
    from circl_b200 import oprf
    s, S = suite
    n = 2 * OP_CHUNK + 77
    info = INFO_MAX
    bnd = edges(msg_chunks(n), Q)
    rng = random.Random(700 + mode)
    ktab = [_sc(rng, s) for _ in range(P if per_op else 1)]
    tab = _inputs_table()
    key = (lambda c: ktab[c % P]) if per_op else (lambda c: ktab[0])
    otab = [om.full_evaluate(s, mode, key(c), tab[c], info) for c in range(Q)]
    idx = np.arange(n) % Q
    K = _rows(ktab)[idx % P] if per_op else _rows(ktab).reshape(-1)
    inputs = [tab[c] for c in idx]
    OUT, ST = _rows(otab)[idx], np.zeros(n, np.uint8)
    kinds = ["long65535", "sk0", "long65534", "skn"] + (["t0"] if mode == 2 else []) if per_op else \
        ["long65535", "long65534"]
    for q, i in enumerate(bnd):
        kind = kinds[q % len(kinds)]
        if kind.startswith("long"):
            inputs[i] = bytes((i + j) & 0xFF for j in range(int(kind[4:])))
        else:
            k = {"sk0": 0, "skn": s.n, "t0": s.n - om.info_scalar(s, info)}[kind]
            K[i] = np.frombuffer(om.i2osp(k, s.Ns), np.uint8)
        sk = K[i].tobytes() if per_op else K.tobytes()
        try:
            OUT[i] = np.frombuffer(om.full_evaluate(s, mode, sk, inputs[i], info), np.uint8)
        except om.OprfError as e:
            ST[i], OUT[i] = e.status, 0
    assert ST.any() == per_op

    def run(keys, msgs):
        try:
            return _np(oprf.FullEvaluateBatch(S, mode, keys, msgs, info)), np.zeros(n, np.uint8)
        except oprf.OprfError as e:
            return _np(e.results), _np(e.status)

    out, st = run(K, inputs)
    _same(st, ST, "host status")
    _same(out, OUT, "host outputs")
    msgs, off = oprf._msgs(inputs)
    dout, dst = run(_cuda(K), (_cuda(msgs), _cuda(off.astype(np.int64))))
    assert np.array_equal(dst, st) and np.array_equal(dout, out)


# ---------------------------------------------------------------- info at its limit
@gpu
def test_info_limits(suite):
    """65535 bytes of info are taken by every entry point; 65536 are refused before any device work, by the C ABI
    (CB200_ERR_ARG, outputs and status bytes untouched, on host and device buffers) and by the Python layer."""
    import torch
    from circl_b200 import _ffi, oprf
    s, S = suite
    Ns, Ne, Nh = s.Ns, s.Ne, S.Nh
    sk, r = om.i2osp(0x1234567, Ns), om.i2osp(0x7654321, Ns)
    el = om.compress(s, om.mul(s, 99, s.g))
    key = oprf.DeriveKey(S, 2, bytes(range(32)), INFO_MAX)
    assert (key.k, key.pub) == om.derive_key(s, 2, bytes(range(32)), INFO_MAX)
    ev, pr = oprf.EvaluateBatch(S, 2, sk, _rows([el]), 1, _rows([r]), INFO_MAX)
    e, proof = om.evaluate(s, 2, sk, [el], r, INFO_MAX)
    assert ev[0].tobytes() == e[0] and pr[0].tobytes() == proof
    out = oprf.FullEvaluateBatch(S, 2, sk, [b"x"], INFO_MAX)
    assert out[0].tobytes() == om.full_evaluate(s, 2, sk, b"x", INFO_MAX)

    over = INFO_MAX + b"!"
    for mode in (0, 1, 2):
        for call in (lambda: oprf.DeriveKeyBatch(S, mode, np.zeros((1, 32), np.uint8), over),
                     lambda: oprf.EvaluateBatch(S, mode, sk, _rows([el]), 1, _rows([r]), over),
                     lambda: oprf.FullEvaluateBatch(S, mode, sk, [b"x"], over)):
            with pytest.raises(oprf.ErrInvalidInfo):
                call()
    L = _ffi.lib()
    _ffi.check(L.cb200_set_stream(torch.cuda.current_stream().cuda_stream))
    ibuf = np.frombuffer(over, np.uint8).copy()
    for dev in (False, True):
        def buf(a):
            return _cuda(a) if dev else np.ascontiguousarray(a)

        def p(a):
            return a.data_ptr() if dev else a.ctypes.data

        seeds, K, B, R = buf(np.zeros((2, 32), np.uint8)), buf(_rows([sk, sk])), buf(_rows([el, el])), \
            buf(_rows([r, r]))
        msgs, off = buf(np.frombuffer(b"ab", np.uint8).copy()), buf(np.array([0, 1, 2], np.int64))
        for mode in (0, 1, 2):
            outs = [buf(np.full(shape, 0xA5, np.uint8)) for shape in ((2, Ns), (2, Ne), (2, Ne), (2, 2 * Ns), (2,),
                                                                       (2, Nh), (2,))]
            o = [p(x) for x in outs]
            assert L.cb200_oprf_derive_key(S.id, mode, p(seeds), ibuf.ctypes.data, 65536, o[0], o[1], 2) == \
                CB200_ERR_ARG
            assert L.cb200_oprf_evaluate(S.id, mode, p(K), Ns, p(B), 1, p(R), ibuf.ctypes.data, 65536, o[2], o[3], o[4],
                                         2) == CB200_ERR_ARG
            assert L.cb200_oprf_full_evaluate(S.id, mode, p(K), Ns, p(msgs), p(off), ibuf.ctypes.data, 65536, o[5],
                                              o[6], 2) == CB200_ERR_ARG
            if dev:
                torch.cuda.synchronize()
            for x in outs:
                assert (_np(x) == 0xA5).all()


# ---------------------------------------------------------------- per-op keys inside wider rows
@gpu
def test_strided_keys_through_the_c_abi(suite):
    """Per-op keys at sk_stride = Ns + 5, the padding filled with 0xA5: host buffers across chunks (the 2-D staging
    copy) and device buffers, for Evaluate (mode 1, m = 8) and FullEvaluate (mode 2)."""
    import torch
    from circl_b200 import _ffi, oprf
    s, S = suite
    L = _ffi.lib()
    _ffi.check(L.cb200_set_stream(torch.cuda.current_stream().cuda_stream))
    Ns, W = s.Ns, s.Ns + 5

    def wide(K):
        w = np.full((K.shape[0], W), 0xA5, np.uint8)
        w[:, :Ns] = K
        return w

    def p(a):
        return a.data_ptr() if hasattr(a, "data_ptr") else a.ctypes.data

    m, n = 8, 2 * 4096 + 37
    b = EvalBatch(s, 1, m, n, True, b"", 800, edges(staged(n, eval_chunk(m))))
    Kw = wide(b.K)
    for dev in (False, True):
        K, B, R = [_cuda(a) if dev else a for a in (Kw, b.B, b.R)]
        ev, pr, st = [_cuda(np.zeros(a.shape, np.uint8)) if dev else np.zeros(a.shape, np.uint8)
                      for a in (b.EV, b.PR, b.ST)]
        _ffi.check(L.cb200_oprf_evaluate(S.id, 1, p(K), W, p(B), m, p(R), None, 0, p(ev), p(pr), p(st), n))
        torch.cuda.synchronize()
        b.check((_np(ev), _np(pr), _np(st)), "device" if dev else "host")

    n = OP_CHUNK + 77
    info = b"strided"
    rng = random.Random(801)
    ktab, tab = [_sc(rng, s) for _ in range(P)], _inputs_table()
    otab = [om.full_evaluate(s, 2, ktab[c % P], tab[c], info) for c in range(Q)]
    idx = np.arange(n) % Q
    Kn, OUT, ST = _rows(ktab)[idx % P], _rows(otab)[idx], np.zeros(n, np.uint8)
    for q, i in enumerate(edges(msg_chunks(n), Q)):
        Kn[i] = np.frombuffer(om.i2osp([0, s.n, s.n - om.info_scalar(s, info)][q % 3], Ns), np.uint8)
        with pytest.raises(om.OprfError) as e:
            om.full_evaluate(s, 2, Kn[i].tobytes(), tab[i % Q], info)
        ST[i], OUT[i] = e.value.status, 0
    msgs, off = oprf._msgs([tab[c] for c in idx])
    for dev in (False, True):
        K, M, O = [_cuda(a) if dev else a for a in (wide(Kn), msgs, off.astype(np.int64))]
        out, st = [_cuda(np.zeros(a.shape, np.uint8)) if dev else np.zeros(a.shape, np.uint8) for a in (OUT, ST)]
        _ffi.check(L.cb200_oprf_full_evaluate(S.id, 2, p(K), W, p(M), p(O), info, len(info), p(out), p(st), n))
        torch.cuda.synchronize()
        _same(_np(st), ST, "status")
        _same(_np(out), OUT, "outputs")
