"""The OPRF servers on the GPU, per suite and mode, against the reference's RFC 9497 vectors and tests/oprf_model.py:
every NIST-suite vector through the C ABI (DeriveKey, Evaluate with m = 1 and 2 and its proof, FullEvaluate); seeded
random batches of 2^10 requests with m = 1 and 3, under one shared key and under per-op keys, on host and CUDA buffers;
a round trip with the model as the client; invalid inputs inside valid batches, each failing only its own op; device
rows at odd byte offsets; and a host batch split across GPUs."""
import numpy as np
import pytest

import oprf_model as om
from conftest import load_golden

pytestmark = pytest.mark.gpu

IDENT = ["P256-SHA256", "P384-SHA384", "P521-SHA512"]


@pytest.fixture(scope="module")
def cb():
    import circl_b200
    circl_b200.init(0)
    yield circl_b200
    circl_b200.shutdown()


@pytest.fixture(params=IDENT, ids=["p256", "p384", "p521"])
def suite(request, cb):
    from circl_b200 import oprf
    return om.SUITES[request.param], oprf.GetSuite(request.param)


def _pmap(fn, *cols):
    """fn over the sampled rows (the model is pure Python and fast enough for a few dozen)."""
    return list(map(fn, *cols))


def _u8(b: bytes, rows=1):
    return np.frombuffer(bytes(b), dtype=np.uint8).reshape(rows, -1).copy()


def _x(h):
    return bytes.fromhex(h)


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_rfc9497_vectors_through_the_c_abi(suite, mode):
    from circl_b200 import oprf
    s, S = suite
    tv = next(v for v in load_golden("oprf_rfc9497.json.gz") if v["identifier"] == s.identifier and v["mode"] == mode)
    key = oprf.DeriveKey(S, mode, _x(tv["seed"]), _x(tv["keyInfo"]))
    assert key.k.hex() == tv["skSm"]
    if "pkSm" in tv:
        assert key.Public().MarshalBinary().hex() == tv["pkSm"]
    srv = [oprf.NewServer, oprf.NewVerifiableServer, oprf.NewPartialObliviousServer][mode](S, key)
    for v in tv["vectors"]:
        info = _x(v.get("Info", ""))
        blinded = [_x(h) for h in v["BlindedElement"].split(",")]
        r = _x(v["Proof"]["r"]) if "Proof" in v else None
        ev, proof = srv.Evaluate(blinded, info, r) if mode == 2 else srv.Evaluate(blinded, r)
        assert [e.hex() for e in ev] == v["EvaluationElement"].split(",")
        assert (proof.hex() if proof else None) == (v["Proof"]["proof"] if "Proof" in v else None)
        for inp, out in zip(v["Input"].split(","), v["Output"].split(",")):
            got = srv.FullEvaluate(_x(inp), info) if mode == 2 else srv.FullEvaluate(_x(inp))
            assert got.hex() == out
            args = (_x(inp), info) if mode == 2 else (_x(inp),)
            assert srv.VerifyFinalize(*args, _x(out))
            assert not srv.VerifyFinalize(*args, bytes(len(_x(out))))


def _model_eval(args):
    ident, mode, sk, bl, r, info = args
    s = om.SUITES[ident]
    ev, proof = om.evaluate(s, mode, sk, bl, r, info)
    return b"".join(ev), proof


def _model_full(args):
    ident, mode, sk, inp, info = args
    return om.full_evaluate(om.SUITES[ident], mode, sk, inp, info)


def _batch(s, n, m, seed, shared):
    rng = np.random.default_rng(seed)
    nk = 1 if shared else n
    sks = [om.i2osp(int.from_bytes(rng.bytes(s.Ns + 8), "big") % (s.n - 1) + 1, s.Ns) for _ in range(nk)]
    rs = [om.i2osp(int.from_bytes(rng.bytes(s.Ns + 8), "big") % (s.n - 1) + 1, s.Ns) for _ in range(n)]
    base = [om.compress(s, om.mul(s, int(rng.integers(1, 2**62)), s.g)) for _ in range(8)]
    bl = [[base[int(rng.integers(8))] for _ in range(m)] for _ in range(n)]
    inputs = [rng.bytes(int(rng.integers(0, 200))) for _ in range(n)]
    return sks, rs, bl, inputs


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("m,shared", [(1, True), (3, False)])
def test_model_parity(suite, mode, m, shared):
    import torch
    from circl_b200 import oprf
    s, S = suite
    n = 1 << 10
    sks, rs, bl, inputs = _batch(s, n, m, 7 + mode + m, shared)
    info = b"info for the batch" if mode == 2 else b""
    skarr = _u8(sks[0]).reshape(-1) if shared else _u8(b"".join(sks), n)
    B = _u8(b"".join(b"".join(x) for x in bl), n)
    R = _u8(b"".join(rs), n)
    ev, proof = oprf.EvaluateBatch(S, mode, skarr, B, m, R if mode else None, info)
    out = oprf.FullEvaluateBatch(S, mode, skarr, inputs, info)
    idx = list(range(0, n, 37)) + [n - 1]
    key = lambda i: sks[0] if shared else sks[i]  # noqa: E731
    want = _pmap(_model_eval, [(s.identifier, mode, key(i), bl[i], rs[i] if mode else None, info) for i in idx])
    wout = _pmap(_model_full, [(s.identifier, mode, key(i), inputs[i], info) for i in idx])
    for i, (e, p), o in zip(idx, want, wout):
        assert ev[i].tobytes() == e, i
        assert (proof[i].tobytes() if mode else None) == p, i
        assert out[i].tobytes() == o, i
    # the same on CUDA buffers
    dsk = torch.from_numpy(skarr).cuda()
    dev, dproof = oprf.EvaluateBatch(S, mode, dsk, torch.from_numpy(B).cuda(), m,
                                     torch.from_numpy(R).cuda() if mode else None, info)
    assert np.array_equal(dev.cpu().numpy(), ev)
    if mode:
        assert np.array_equal(dproof.cpu().numpy(), proof)
    msgs, off = oprf._msgs(inputs)
    dout = oprf.FullEvaluateBatch(S, mode, dsk, (torch.from_numpy(msgs).cuda(),
                                                 torch.from_numpy(off.astype(np.int64)).cuda()), info)
    assert np.array_equal(dout.cpu().numpy(), out)


@pytest.mark.parametrize("mode", [1, 2])
def test_round_trip_with_the_model_client(suite, mode):
    from circl_b200 import oprf
    s, S = suite
    key = oprf.DeriveKey(S, mode, bytes(range(32)), b"round trip")
    srv = (oprf.NewVerifiableServer if mode == 1 else oprf.NewPartialObliviousServer)(S, key)
    info = b"public info" if mode == 2 else b""
    inputs = [b"", b"a", bytes(range(100))]
    blinds = [12345 + i for i in range(3)]
    bl = [om.blind(s, mode, x, b) for x, b in zip(inputs, blinds)]
    ev, proof = srv.Evaluate(bl, info) if mode == 2 else srv.Evaluate(bl)
    assert om.client_verify(s, mode, key.Public().MarshalBinary(), bl, ev, proof, info)
    for x, b, e in zip(inputs, blinds, ev):
        out = om.finalize(s, mode, x, b, e, info)
        got = srv.FullEvaluate(x, info) if mode == 2 else srv.FullEvaluate(x)
        assert got == out
        assert srv.VerifyFinalize(*((x, info) if mode == 2 else (x,)), out)


def test_invalid_inputs_fail_only_their_own_op(suite):
    import torch
    from circl_b200 import oprf
    s, S = suite
    n, m, Ne, Ns = 16, 2, s.Ne, s.Ns
    sks, rs, bl, _ = _batch(s, n, m, 99, False)
    x = next(v for v in range(1, 200) if not om._is_square(s, (v ** 3 - 3 * v + s.b) % s.p))
    bad_el = {1: b"\x04" + bl[1][0][1:], 2: b"\x02" + om.i2osp(s.p, s.nbytes), 3: b"\x03" + om.i2osp(x, s.nbytes)}
    for i, e in bad_el.items():
        bl[i][1] = e
    sks[4] = bytes(Ns)
    sks[5] = om.i2osp(s.n, Ns)
    rs[6] = bytes(Ns)
    rs[7] = om.i2osp(s.n + 1, Ns) if s.n + 1 < 2**(8 * Ns) else b"\xff" * Ns
    info = b"t = 0 here"
    sks[8] = om.i2osp(s.n - om.info_scalar(s, info), Ns)
    want = {1: 1, 2: 1, 3: 1, 4: 2, 5: 2, 6: 4, 7: 4}
    B = _u8(b"".join(b"".join(x) for x in bl), n)
    K, R = _u8(b"".join(sks), n), _u8(b"".join(rs), n)
    for mode in (1, 2):
        w = dict(want)
        if mode == 2:
            w[8] = 8
        for dev in (False, True):
            args = [torch.from_numpy(a).cuda() if dev else a for a in (K, B, R)]
            with pytest.raises(oprf.OprfError) as ei:
                oprf.EvaluateBatch(S, mode, args[0], args[1], m, args[2], info if mode == 2 else b"")
            st = ei.value.status.cpu().numpy() if dev else ei.value.status
            ev, proof = [t.cpu().numpy() if dev else t for t in ei.value.results]
            assert {i: int(v) for i, v in enumerate(st) if v} == w
            for i in range(n):
                if i in w:
                    assert not ev[i].any() and not proof[i].any()
                else:
                    e, p = om.evaluate(s, mode, sks[i], bl[i], rs[i], info if mode == 2 else b"")
                    assert ev[i].tobytes() == b"".join(e) and proof[i].tobytes() == p
    # shared keys: 0 and n fail every op, in Evaluate (every mode, host and CUDA buffers) and in FullEvaluate
    good = _u8(b"".join(b"".join(x) for x in bl[9:12]), 3)
    for bad in (bytes(Ns), om.i2osp(s.n, Ns)):
        for mode in (0, 1, 2):
            for dev in (False, True):
                k, b_, r_ = [torch.from_numpy(a).cuda() if dev else a for a in (_u8(bad).reshape(-1), good, R[9:12])]
                with pytest.raises(oprf.ErrInvalidPrivateKey) as ei:
                    oprf.EvaluateBatch(S, mode, k, b_, m, r_ if mode else None, b"i")
                st = ei.value.status.cpu().numpy() if dev else ei.value.status
                assert list(st) == [2, 2, 2]
                for t in ei.value.results:
                    if t is not None:
                        assert not (t.cpu().numpy() if dev else t).any()
        with pytest.raises(oprf.ErrInvalidPrivateKey) as ei:
            oprf.FullEvaluateBatch(S, 0, _u8(bad).reshape(-1), [b"x", b"y"])
        assert list(ei.value.status) == [2, 2]


def test_device_rows_at_odd_offsets(suite):
    import torch
    from circl_b200 import oprf
    s, S = suite
    n, Ne, Ns = 33, s.Ne, s.Ns
    sks, rs, bl, inputs = _batch(s, n, 1, 5, False)
    B, K, R = _u8(b"".join(x[0] for x in bl), n), _u8(b"".join(sks), n), _u8(b"".join(rs), n)
    ev, proof = oprf.EvaluateBatch(S, 1, K, B, 1, R)
    out = oprf.FullEvaluateBatch(S, 1, K, inputs)
    from circl_b200 import _ffi
    L = _ffi.lib()
    buf = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    o = [1, 3 + n * Ns, 5 + 2 * n * Ns, 7 + 3 * n * Ns + n * Ne, 9 + 3 * n * Ns + 2 * n * Ne,
         11 + 3 * n * Ns + 2 * n * Ne + n * 2 * Ns]
    for a, at in ((K, o[0]), (R, o[1]), (B, o[3])):
        buf[at:at + a.size] = torch.from_numpy(a.reshape(-1)).cuda()
    p = buf.data_ptr()
    _ffi.check(L.cb200_set_stream(torch.cuda.current_stream().cuda_stream))
    _ffi.check(L.cb200_oprf_evaluate(S.id, 1, p + o[0], Ns, p + o[3], 1, p + o[1], None, 0, p + o[4], p + o[5],
                                     p + o[2], n))
    torch.cuda.synchronize()
    h = buf.cpu().numpy()
    assert np.array_equal(h[o[4]:o[4] + n * Ne].reshape(n, Ne), ev)
    assert np.array_equal(h[o[5]:o[5] + n * 2 * Ns].reshape(n, 2 * Ns), proof)
    assert not h[o[2]:o[2] + n].any()
    # FullEvaluate with sk, the inputs, the outputs and the status bytes at odd offsets (msg_off 8-byte aligned)
    msgs, off = oprf._msgs(inputs)
    buf.zero_()
    Nh = S.Nh
    q = [1, 3 + n * Ns, 8 * ((5 + n * Ns + msgs.size) // 8 + 1)]
    q += [q[2] + 8 * (n + 1) + 3, q[2] + 8 * (n + 1) + 5 + n * Nh]
    buf[q[0]:q[0] + K.size] = torch.from_numpy(K.reshape(-1)).cuda()
    buf[q[1]:q[1] + msgs.size] = torch.from_numpy(msgs).cuda()
    buf[q[2]:q[2] + 8 * (n + 1)] = torch.from_numpy(off.view(np.uint8)).cuda()
    _ffi.check(L.cb200_oprf_full_evaluate(S.id, 1, p + q[0], Ns, p + q[1], p + q[2], None, 0, p + q[3], p + q[4], n))
    torch.cuda.synchronize()
    h = buf.cpu().numpy()
    assert np.array_equal(h[q[3]:q[3] + n * Nh].reshape(n, Nh), out)
    assert not h[q[4]:q[4] + n].any()


def test_device_input_over_65535_bytes_fails_its_own_op(suite):
    """A device-pointer FullEvaluate cannot refuse the call on an input length it does not read: the op gets status 16
    and a zero output, its neighbours are unaffected.  The host-pointer call refuses it before any device work."""
    import torch
    from circl_b200 import oprf
    s, S = suite
    sk = om.i2osp(12345, s.Ns)
    inputs = [b"a", bytes(65535), bytes(65536), b"b"]
    big = np.frombuffer(b"".join(inputs), dtype=np.uint8).copy()
    off = np.cumsum([0] + [len(x) for x in inputs]).astype(np.int64)
    with pytest.raises(oprf.ErrInvalidInput) as ei:
        oprf.FullEvaluateBatch(S, 0, _u8(sk).reshape(-1), (torch.from_numpy(big).cuda(), torch.from_numpy(off).cuda()))
    assert list(ei.value.status.cpu().numpy()) == [0, 0, 16, 0]
    out = ei.value.results.cpu().numpy()
    assert not out[2].any()
    for i in (0, 1, 3):
        assert out[i].tobytes() == om.full_evaluate(s, 0, sk, inputs[i])
    with pytest.raises(oprf.ErrInvalidInput):
        oprf.FullEvaluateBatch(S, 0, _u8(sk).reshape(-1), inputs)


@pytest.mark.parametrize("ident", IDENT)
def test_host_batch_split_across_gpus(ident):
    import circl_b200
    from circl_b200 import _ffi, oprf
    if _ffi.lib().cb200_device_count() < 2:
        pytest.skip("needs two GPUs")
    circl_b200.init_devices(0)
    try:
        s, S = om.SUITES[ident], oprf.GetSuite(ident)
        n = (1 << 13) + 11
        sks, rs, bl, inputs = _batch(s, n, 1, 41, True)
        B, R = _u8(b"".join(x[0] for x in bl), n), _u8(b"".join(rs), n)
        ev, proof = oprf.EvaluateBatch(S, 1, _u8(sks[0]).reshape(-1), B, 1, R)
        out = oprf.FullEvaluateBatch(S, 1, _u8(sks[0]).reshape(-1), inputs)
        for i in (0, n // 2 - 1, n // 2, n - 1):
            e, p = om.evaluate(s, 1, sks[0], bl[i], rs[i])
            assert ev[i].tobytes() == e[0] and proof[i].tobytes() == p
            assert out[i].tobytes() == om.full_evaluate(s, 1, sks[0], inputs[i])
    finally:
        circl_b200.shutdown()
