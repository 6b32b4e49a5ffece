"""CPU-only: the Prio3 entry points are exported, cb200_prio3_get_sizes gives the model's wire sizes for every vector
file's configuration, every configuration error the reference's New returns (and ErrAggID, null pointers, a work area
over the bound) is CB200_ERR_ARG before the device is touched, and valid calls fail loudly without a device."""
import ctypes as C

import numpy as np
import pytest

import prio3_model as M
from conftest import load_golden


def _cfg(kind, shares=2, ctx=b"", **kw):
    from circl_b200 import prio3
    c = prio3._Config(kind=kind, num_shares=shares, context=ctx, context_len=len(ctx), **kw)
    c._keep = ctx
    return c


def _sizes(c):
    from circl_b200 import _ffi, prio3
    z = prio3._Sizes()
    rc = _ffi.lib().cb200_prio3_get_sizes(C.byref(c), C.byref(z))
    return rc, {k: getattr(z, k) for k, _ in prio3._Sizes._fields_}


def test_exports():
    from circl_b200._ffi import lib
    L = C.CDLL(lib()._name)
    for name in ("get_sizes", "prep_init", "prep_shares_to_prep", "prep_next", "aggregate"):
        assert hasattr(L, "cb200_prio3_" + name), name


@pytest.mark.parametrize("name", M.VECTOR_FILES)
def test_sizes_of_vector_configs(name):
    from circl_b200 import prio3
    v = load_golden("prio3_%s.json.gz" % name)
    P = M.from_vector(name, v)
    ctx = bytes.fromhex(v["ctx"])
    kw = {"Count": {}, "Sum": dict(max_measurement=v.get("max_measurement", 0)),
          "SumVec": dict(length=v.get("length", 0), bits=v.get("bits", 0), chunk_length=v.get("chunk_length", 0)),
          "Histogram": dict(length=v.get("length", 0), chunk_length=v.get("chunk_length", 0)),
          "MultihotCountVec": dict(length=v.get("length", 0), max_weight=v.get("max_weight", 0),
                                   chunk_length=v.get("chunk_length", 0))}[name.split("_")[0]]
    rc, z = _sizes(_cfg(P.c.ID, v["shares"], ctx, **kw))
    assert rc == 0 and z == P.sizes()
    r = v["prep"][0]
    assert z["input_share_leader"] * 2 == len(r["input_shares"][0])
    assert z["input_share_helper"] * 2 == len(r["input_shares"][1])
    assert z["prep_share"] * 2 == len(r["prep_shares"][0][0])
    # the Python classes report the same sizes
    cls = {1: prio3.Count, 2: prio3.Sum, 3: prio3.SumVec, 4: prio3.Histogram, 5: prio3.MultiHotCountVec}[P.c.ID]
    args = {1: (), 2: (kw.get("max_measurement"),), 3: (kw.get("length"), kw.get("bits"), kw.get("chunk_length")),
            4: (kw.get("length"), kw.get("chunk_length")),
            5: (kw.get("length"), kw.get("max_weight"), kw.get("chunk_length"))}[P.c.ID]
    assert cls(v["shares"], *args, ctx).Params() == z


BAD = [
    ("numshares 1", dict(kind=1, shares=1)),
    ("numshares 256", dict(kind=1, shares=256)),
    ("unknown kind", dict(kind=6)),
    ("kind 0", dict(kind=0)),
    ("context too long", dict(kind=1, ctx=bytes(65528))),
    ("sum max >= 2^63", dict(kind=2, max_measurement=1 << 63)),
    ("sumvec length 0", dict(kind=3, length=0, bits=1, chunk_length=1)),
    ("sumvec bits 0", dict(kind=3, length=1, bits=0, chunk_length=1)),
    ("sumvec bits 65", dict(kind=3, length=1, bits=65, chunk_length=1)),
    ("sumvec chunk 0", dict(kind=3, length=1, bits=1, chunk_length=0)),
    ("histogram length 0", dict(kind=4, length=0, chunk_length=1)),
    ("histogram chunk 0", dict(kind=4, length=1, chunk_length=0)),
    ("mhcv length 0", dict(kind=5, length=0, max_weight=0, chunk_length=1)),
    ("mhcv weight > length", dict(kind=5, length=3, max_weight=4, chunk_length=1)),
    ("mhcv chunk 0", dict(kind=5, length=3, max_weight=1, chunk_length=0)),
    ("work area", dict(kind=4, length=1 << 23, chunk_length=1 << 23)),
    # lengths past 32 bits: refused on their 64-bit values, not after narrowing
    ("histogram length 2^32", dict(kind=4, length=(1 << 32) + 10, chunk_length=(1 << 32) + 10)),
    ("sumvec length 2^32", dict(kind=3, length=1 << 32, bits=1, chunk_length=1 << 32)),
    ("mhcv length 2^32", dict(kind=5, length=1 << 32, max_weight=1, chunk_length=1 << 32)),
]


@pytest.mark.parametrize("what,kw", BAD, ids=[b[0] for b in BAD])
def test_config_errors(what, kw):
    from circl_b200 import _ffi
    kind, shares, ctx = kw.pop("kind"), kw.pop("shares", 2), kw.pop("ctx", b"")
    c = _cfg(kind, shares, ctx, **kw)
    rc, _ = _sizes(c)
    assert rc == -1
    L = _ffi.lib()
    z = np.zeros(1 << 16, np.uint8)
    p = z.ctypes.data
    assert L.cb200_prio3_prep_init(C.byref(c), p, 0, p, p, p, p, p, p, 1) == -1
    assert L.cb200_prio3_prep_shares_to_prep(C.byref(c), p, p, p, 1) == -1
    assert L.cb200_prio3_prep_next(C.byref(c), p, p, p, p, 1) == -1
    assert L.cb200_prio3_aggregate(C.byref(c), p, p, p, 1) == -1


def test_call_errors_and_no_device():
    from circl_b200 import _ffi
    L = _ffi.lib()
    z = np.zeros(1 << 16, np.uint8)
    p = z.ctypes.data
    cnt, hist = _cfg(1), _cfg(4, 3, b"x", length=10, chunk_length=3)
    from circl_b200 import prio3
    assert L.cb200_prio3_get_sizes(None, C.byref(prio3._Sizes())) == -1
    assert L.cb200_prio3_get_sizes(C.byref(cnt), None) == -1
    assert L.cb200_prio3_prep_init(C.byref(cnt), p, 2, p, None, p, p, p, p, 1) == -1  # ErrAggID
    assert L.cb200_prio3_prep_init(C.byref(hist), p, 3, p, p, p, p, p, p, 1) == -1
    assert L.cb200_prio3_prep_init(C.byref(hist), p, 1, p, None, p, p, p, p, 1) == -1  # public share required
    assert L.cb200_prio3_prep_init(C.byref(cnt), None, 0, p, None, p, p, p, p, 1) == -1
    assert L.cb200_prio3_prep_shares_to_prep(C.byref(hist), p, None, p, 1) == -1
    assert L.cb200_prio3_prep_next(C.byref(cnt), p, None, p, None, 1) == -1
    assert L.cb200_prio3_aggregate(C.byref(cnt), None, None, p, 1) == -1
    # valid calls without a device
    assert L.cb200_prio3_prep_init(C.byref(cnt), p, 1, p, None, p, p, p, p, 1) == -2
    assert L.cb200_prio3_prep_init(C.byref(hist), p, 2, p, p, p, p, p, p, 1) == -2
    assert L.cb200_prio3_prep_shares_to_prep(C.byref(hist), p, p, p, 1) == -2
    assert L.cb200_prio3_prep_next(C.byref(cnt), p, None, p, p, 1) == -2
    assert L.cb200_prio3_aggregate(C.byref(hist), p, None, p, 1) == -2


def test_python_errors():
    from circl_b200 import prio3
    for f in (lambda: prio3.Count(1), lambda: prio3.Sum(2, 1 << 63), lambda: prio3.SumVec(2, 1, 65, 1),
              lambda: prio3.Histogram(2, 0, 1), lambda: prio3.MultiHotCountVec(2, 3, 4, 1),
              lambda: prio3.Count(2, bytes(65528))):
        with pytest.raises(ValueError):
            f()
    h = prio3.Histogram(2, 4, 2)
    assert h.Unshard([h.AggregateInit(), h.AggregateUpdate(h.AggregateInit(), (1).to_bytes(16, "little") * 4)], 1) \
        == [1, 1, 1, 1]
    s = prio3.Sum(2, 2**32)
    with pytest.raises(ValueError):
        s.Unshard([s.AggregateInit()] * 2, 2**32)
