"""Prio3 aggregators on the GPU through the C ABI and circl_b200.prio3, against the reference's vectors and
tests/prio3_model.py:
  - every vector file and aggregator: PrepInit -> prep shares, PrepSharesToPrep -> prep messages, PrepNext -> out
    shares, Aggregate -> agg shares, Unshard -> the aggregate result; on host buffers and on CUDA tensors;
  - random reports from the model's Shard, 2 and 3 shares, leader and helpers, for every circuit, including a Histogram
    of length 1000 and a SumVec whose domain is larger than a warp;
  - invalid reports failing only their own rows, each at its own step, and left out of Aggregate;
  - device rows at odd byte offsets;
  - a host batch past one staging chunk, with Aggregate equal to the sum of its parts."""
import concurrent.futures as cf
import os
import random

import numpy as np
import pytest

import prio3_model as M
from conftest import load_golden

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def runtime():
    import circl_b200
    circl_b200.init(0)
    yield


def _cls(P):
    from circl_b200 import prio3
    c = P.c
    if c.ID == 1:
        return prio3.Count(P.shares, P.ctx)
    if c.ID == 2:
        return prio3.Sum(P.shares, c.max, P.ctx)
    if c.ID == 3:
        return prio3.SumVec(P.shares, c.length, c.bits, c.chunk, P.ctx)
    if c.ID == 4:
        return prio3.Histogram(P.shares, c.length, c.chunk, P.ctx)
    return prio3.MultiHotCountVec(P.shares, c.length, 2**c.bits - 1 - c.offset, c.chunk, P.ctx)


def _arr(rows, width):
    return np.frombuffer(b"".join(rows), np.uint8).reshape(len(rows), width) if width else None


def _to(x, dev):
    if x is None or not dev:
        return x
    import torch
    return torch.from_numpy(np.array(x)).cuda()


def _np(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else x


def run_all(V, vk, nonces, pubs, ins, dev=False):
    """PrepInit for every aggregator, PrepSharesToPrep, PrepNext, Aggregate over n reports; returns numpy results"""
    z = V.Params()
    n = len(nonces)
    states, shares, st_init = [], [], []
    for a in range(V.shares):
        w = z["input_share_helper" if a else "input_share_leader"]
        s, h, st = V.PrepInitBatch(vk, a, _to(_arr(nonces, 16), dev), _to(_arr(pubs, z["public_share"]), dev),
                                   _to(_arr([r[a] for r in ins], w), dev))
        states.append(_np(s))
        shares.append(_np(h))
        st_init.append(_np(st))
    rows = np.concatenate(shares, axis=1)
    msgs, st_dec = V.PrepSharesToPrepBatch(_to(rows, dev))
    msgs, st_dec = _np(msgs), _np(st_dec)
    outs, st_next, aggs = [], [], []
    for a in range(V.shares):
        o, st = V.PrepNextBatch(_to(states[a], dev), _to(msgs, dev) if z["prep_msg"] else None)
        o, st = _np(o), _np(st)
        ok = (st | st_dec | st_init[a]).astype(np.uint8)
        agg = V.AggregateBatch(_to(o, dev), _to(ok, dev))
        aggs.append(bytes(_np(agg).tobytes()) if dev else agg)
        outs.append(o)
        st_next.append(st)
    return dict(states=states, shares=shares, st_init=st_init, msgs=msgs, st_dec=st_dec, outs=outs, st_next=st_next,
                aggs=aggs)


@pytest.mark.parametrize("dev", [False, True], ids=["host", "cuda"])
@pytest.mark.parametrize("name", M.VECTOR_FILES)
def test_vectors(name, dev):
    v = load_golden("prio3_%s.json.gz" % name)
    P = M.from_vector(name, v)
    V = _cls(P)
    assert V.Params() == P.sizes()
    prep = v["prep"]
    r = run_all(V, bytes.fromhex(v["verify_key"]), [bytes.fromhex(p["nonce"]) for p in prep],
                [bytes.fromhex(p["public_share"]) for p in prep],
                [[bytes.fromhex(s) for s in p["input_shares"]] for p in prep], dev)
    for i, p in enumerate(prep):
        assert [r["shares"][a][i].tobytes().hex() for a in range(P.shares)] == p["prep_shares"][0]
        assert r["msgs"][i].tobytes().hex() == p["prep_messages"][0]
        assert [r["outs"][a][i].tobytes().hex() for a in range(P.shares)] == ["".join(o) for o in p["out_shares"]]
    assert not any(s.any() for s in r["st_init"] + r["st_next"]) and not r["st_dec"].any()
    assert [a.hex() for a in r["aggs"]] == v["agg_shares"]
    assert V.Unshard(r["aggs"], len(prep)) == v["agg_result"]
    # the per-report methods
    p = prep[0]
    nonce, pub = bytes.fromhex(p["nonce"]), bytes.fromhex(p["public_share"])
    got = [V.PrepInit(bytes.fromhex(v["verify_key"]), nonce, a, pub, bytes.fromhex(p["input_shares"][a]))
           for a in range(P.shares)]
    msg = V.PrepSharesToPrep([g[1] for g in got])
    assert msg.hex() == p["prep_messages"][0]
    assert V.PrepNext(got[0][0], msg).hex() == "".join(p["out_shares"][0])


def _shard_one(args):
    mk, shares, ctx, seed, meas = args
    rng = random.Random(seed)
    P = M.Prio3(mk(), shares, ctx)
    nonce = rng.randbytes(16)
    pub, ins = P.shard(meas, nonce, rng.randbytes(P.rand_size()))
    return nonce, pub, ins


def _pmap(fn, items):
    with cf.ProcessPoolExecutor(max_workers=min(16, os.cpu_count() or 1)) as ex:
        return list(ex.map(fn, items, chunksize=max(1, len(items) // 64)))


def _model_check(P, vk, nonces, pubs, ins, r, idx):
    """the model's PrepInit / PrepSharesToPrep / PrepNext on rows idx equal the device's"""
    for i in idx:
        shares = []
        for a in range(P.shares):
            st, state, share = P.prep_init(vk, a, nonces[i], pubs[i], ins[i][a])
            assert (st, state, share) == (int(r["st_init"][a][i]), r["states"][a][i].tobytes(),
                                          r["shares"][a][i].tobytes())
            shares.append(share)
        st, msg = P.prep_shares_to_prep(shares)
        assert (st, msg) == (int(r["st_dec"][i]), r["msgs"][i].tobytes())


class _Hist:  # picklable constructors for the process pool
    def __init__(self, *a):
        self.a = a

    def __call__(self):
        return M.Histogram(*self.a)


class _SumVec(_Hist):
    def __call__(self):
        return M.SumVec(*self.a)


class _Mhcv(_Hist):
    def __call__(self):
        return M.MultiHotCountVec(*self.a)


class _Sum(_Hist):
    def __call__(self):
        return M.Sum(*self.a)


class _Count(_Hist):
    def __call__(self):
        return M.Count()


def _hot(rng, length, weight):
    on = set(rng.sample(range(length), weight))
    return [i in on for i in range(length)]


RANDOM = [
    ("count", _Count(), 3000, lambda rng: rng.randrange(2)),
    ("sum", _Sum(2**16 - 1), 2000, lambda rng: rng.randrange(2**16)),
    ("histogram100", _Hist(100, 10), 200, lambda rng: rng.randrange(100)),
    ("histogram1000", _Hist(1000, 30), 40, lambda rng: rng.randrange(1000)),
    ("sumvec", _SumVec(100, 8, 12), 100, lambda rng: [rng.randrange(256) for _ in range(100)]),
    ("mhcv", _Mhcv(100, 10, 9), 150, lambda rng: _hot(rng, 100, rng.randrange(11))),
]


@pytest.mark.parametrize("shares", [2, 3])
@pytest.mark.parametrize("name,mk,n,meas", RANDOM, ids=[c[0] for c in RANDOM])
def test_random_reports(name, mk, n, meas, shares):
    rng = random.Random(name + str(shares))
    ctx = b"task " + name.encode()
    P = M.Prio3(mk(), shares, ctx)
    ms = [meas(rng) for _ in range(n)]
    rows = _pmap(_shard_one, [(mk, shares, ctx, "%s-%d-%d" % (name, shares, i), m) for i, m in enumerate(ms)])
    nonces, pubs, ins = [r[0] for r in rows], [r[1] for r in rows], [r[2] for r in rows]
    vk = rng.randbytes(32)
    V = _cls(P)
    r = run_all(V, vk, nonces, pubs, ins)
    assert not any(s.any() for s in r["st_init"] + r["st_next"]) and not r["st_dec"].any()
    _model_check(P, vk, nonces, pubs, ins, r, rng.sample(range(n), min(n, 6)))
    got = V.Unshard(r["aggs"], n)
    if isinstance(ms[0], list):
        want = [sum(int(m[j]) for m in ms) for j in range(len(ms[0]))]
    else:
        want = sum(ms) if name.startswith(("count", "sum")) else [sum(1 for m in ms if m == j) for j in range(P.c.length)]
    assert got == want


INVALID = [
    ("count", _Count(), [1, 0, 2, 1]),
    ("histogram", _Hist(8, 3), [3, 0, 5, 7]),
    ("mhcv", _Mhcv(8, 2, 3), [[1, 0, 0, 0, 0, 0, 0, 1], [0] * 8, [1, 1, 1, 0, 0, 0, 0, 0], [0, 1] + [0] * 6]),
    ("sum", _Sum(100), [5, 100, 7, 0]),
]


def _encode_bad(P, name, m):
    """an encoded measurement outside the circuit: Count 2, a Histogram with two ones, an MHCV over its weight, Sum
    bits that do not encode the value"""
    c = P.c
    if name == "count":
        return [m]
    if name == "histogram":
        return [1 if i in (m, (m + 1) % c.length) else 0 for i in range(c.length)]
    if name == "mhcv":
        return [int(b) for b in m] + M._split_bits(c.offset + sum(m) - 1, c.bits)  # weight bits do not match
    return M._split_bits(m, c.bits) + M._split_bits((m + c.offset + 1) % (1 << c.bits), c.bits)


@pytest.mark.parametrize("name,mk,ms", INVALID, ids=[c[0] for c in INVALID])
def test_invalid_reports_fail_their_own_rows(name, mk, ms):
    rng = random.Random(name)
    P = M.Prio3(mk(), 2, b"bad")
    F = P.F
    V = _cls(P)
    vk = rng.randbytes(32)
    nonces, pubs, ins = [], [], []
    good = []
    for i in range(24):
        m = ms[i % 4] if i % 4 != 2 or i == 2 else ms[0]  # ms[2] is the invalid measurement: row 2 only
        nonce = rng.randbytes(16)
        rnd = rng.randbytes(P.rand_size())
        if i == 2:  # a measurement outside the circuit, proven honestly
            enc = P.c.encode
            P.c.encode = lambda _m, e=_encode_bad(P, name, m): e
            pub, sh = P.shard(m, nonce, rnd)
            P.c.encode = enc
        else:
            pub, sh = P.shard(m, nonce, rnd)
        sh = list(sh)
        if i == 5:  # a tampered leader proof element
            off = F.size * (P.c.meas_len + 1)
            x = (int.from_bytes(sh[0][off:off + F.size], "little") + 1) % F.p
            sh[0] = sh[0][:off] + x.to_bytes(F.size, "little") + sh[0][off + F.size:]
        if i == 7 and pub:  # a tampered public-share part (the helper's)
            pub = pub[:M.SEED] + bytes([pub[M.SEED] ^ 0x80]) + pub[M.SEED + 1:]
        if i == 11:  # a leader element >= p
            sh[0] = (F.p + 3).to_bytes(F.size, "little") + sh[0][F.size:]
        nonces.append(nonce)
        pubs.append(pub)
        ins.append(sh)
        good.append(i not in (2, 5, 7, 11) or (i == 7 and not pub))
    r = run_all(V, vk, nonces, pubs, ins)
    st_h = r["st_init"][1]
    assert int(r["st_dec"][2]) == 8 and int(r["st_dec"][5]) == 8
    assert int(r["st_init"][0][11]) == 1 and int(r["st_dec"][11]) != 0
    if pubs[7]:
        assert int(st_h[7]) == 2
    for i in range(24):
        if good[i]:
            assert int(r["st_init"][0][i]) == 0 and int(st_h[i]) == 0 and int(r["st_dec"][i]) == 0
    for a in range(2):
        for i in range(24):
            if not good[i]:
                assert not r["outs"][a][i].any() or int(r["st_dec"][i]) != 0
    _model_check(P, vk, nonces, pubs, ins, r, range(24))
    # Aggregate over the good rows only equals the model's
    want = [P.aggregate([r["outs"][a][i].tobytes() for i in range(24) if good[i]]) for a in range(2)]
    assert r["aggs"] == want
    # a wrong joint-rand seed in the prep message fails PrepNext
    if P.jr:
        msgs = r["msgs"].copy()
        msgs[0, 0] ^= 1
        o, st = V.PrepNextBatch(r["states"][0], msgs)
        assert int(st[0]) == 2 and not o[0].any() and (st[1:] == r["st_next"][0][1:]).all()


def test_device_rows_at_odd_offsets():
    import torch
    v = load_golden("prio3_Histogram_1.json.gz")
    P = M.from_vector("Histogram_1", v)
    V = _cls(P)
    z = V.Params()
    p = v["prep"][0]
    vk = bytes.fromhex(v["verify_key"])
    n = 5

    def odd(b, w):
        buf = torch.zeros(n * w + 3, dtype=torch.uint8, device="cuda")
        buf[3:] = torch.from_numpy(np.frombuffer(b * n, np.uint8).copy()).cuda()
        return buf[3:].view(n, w)
    a = 1
    s, h, st = V.PrepInitBatch(vk, a, odd(bytes.fromhex(p["nonce"]), 16), odd(bytes.fromhex(p["public_share"]),
                                                                              z["public_share"]),
                               odd(bytes.fromhex(p["input_shares"][a]), z["input_share_helper"]))
    assert not st.any()
    assert all(h[i].cpu().numpy().tobytes().hex() == p["prep_shares"][0][a] for i in range(n))


def test_large_host_batch_across_chunks():
    """a host batch past one staging chunk, split across every visible GPU (one range per GPU when two or more are
    visible): Aggregate equals the sum of its parts and the model's sum, PrepInit equals the vector's rows"""
    import circl_b200
    circl_b200.shutdown()
    circl_b200.init_devices(0)
    try:
        _large_host_batch()
    finally:
        circl_b200.shutdown()
        circl_b200.init(0)


def _large_host_batch():
    from circl_b200 import prio3
    V = prio3.Count(2)
    rng = np.random.default_rng(7)
    n = (1 << 16) * 3 + 123  # past one Aggregate chunk and past 2^14 rows per GPU
    # out shares are field elements: aggregate random canonical rows, split and whole
    vals = rng.integers(0, 2**63, size=n, dtype=np.uint64)  # below p: canonical Field64 elements
    out = vals.view(np.uint8).reshape(n, 8)
    status = (rng.random(n) < 0.1).astype(np.uint8)
    whole = V.AggregateBatch(out, status)
    parts = [V.AggregateBatch(out[i:i + 20000], status[i:i + 20000]) for i in range(0, n, 20000)]
    assert whole == V._merge(parts)
    want = sum(int(x) for x, s in zip(vals, status) if not s) % M.F64.p
    assert int.from_bytes(whole, "little") == want
    # PrepInit past one staging chunk: every row of a repeated vector report
    v = load_golden("prio3_Count_0.json.gz")
    p = v["prep"][0]
    m = 70000
    V = prio3.Count(2, bytes.fromhex(v["ctx"]))
    s, h, st = V.PrepInitBatch(bytes.fromhex(v["verify_key"]), 1,
                               np.tile(np.frombuffer(bytes.fromhex(p["nonce"]), np.uint8), (m, 1)), None,
                               np.tile(np.frombuffer(bytes.fromhex(p["input_shares"][1]), np.uint8), (m, 1)))
    assert not st.any()
    assert (h == np.frombuffer(bytes.fromhex(p["prep_shares"][0][1]), np.uint8)).all()
