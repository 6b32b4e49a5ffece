"""Prio3 aggregators (draft-irtf-cfrg-vdaf-14) over the C ABI: the reference's vdaf/prio3 packages count, sum, sumvec,
histogram and mhcv, aggregator side.  The client's Shard is not served (one measurement per client, nothing to batch).

  Count(numShares, context), Sum(numShares, maxMeasurement, context),
  SumVec(numShares, length, bits, chunkLength, context), Histogram(numShares, length, chunkLength, context),
  MultiHotCountVec(numShares, length, maxWeight, chunkLength, context)
      .Params()                                            the wire sizes (cb200_prio3_get_sizes)
      .PrepInit, .PrepSharesToPrep, .PrepNext              one report, on bytes (prio3.go:245-403)
      .AggregateInit, .AggregateUpdate, .Unshard           on agg shares as bytes (:408-449; Unshard on the host)
      .PrepInitBatch, .PrepSharesToPrepBatch, .PrepNextBatch, .AggregateBatch
                                                           n reports as (n, width) uint8 rows, numpy or CUDA tensors

Every row is the reference's wire encoding.  A batch returns (outputs, status); a per-report method raises the error of
its status bit: ErrDecode (1, an element >= p), ErrJointRand (2), ErrInvalidEval (4), ErrProofVerify (8), each with
.status.  A configuration the reference's New refuses raises ValueError.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._ffi import check, lib
from .hybrid import _is_torch, _new, _prep, _ptr

__all__ = ["Count", "Sum", "SumVec", "Histogram", "MultiHotCountVec", "Prio3Error", "ErrDecode", "ErrJointRand",
           "ErrInvalidEval", "ErrProofVerify"]

P64 = 2**64 - 2**32 + 1
P128 = 2**128 - 28 * 2**64 + 1


class Prio3Error(ValueError):
    def __init__(self, msg="", status=0):
        super().__init__(msg)
        self.status = status


class ErrDecode(Prio3Error):  # UnmarshalBinary: an element >= p
    pass


class ErrJointRand(Prio3Error):  # prio3.ErrJointRand
    pass


class ErrInvalidEval(Prio3Error):  # flp.ErrInvalidEval: t^p = 1
    pass


class ErrProofVerify(Prio3Error):  # prio3.ErrProofVerify
    pass


_ERRORS = ((1, ErrDecode), (2, ErrJointRand), (4, ErrInvalidEval), (8, ErrProofVerify))


def _raise(st):
    for bit, cls in _ERRORS:
        if st & bit:
            raise cls(cls.__name__, st)


class _Config(C.Structure):
    _fields_ = [("kind", C.c_uint32), ("num_shares", C.c_uint32), ("max_measurement", C.c_uint64),
                ("length", C.c_uint64), ("bits", C.c_uint64), ("chunk_length", C.c_uint64),
                ("max_weight", C.c_uint64), ("context", C.c_char_p), ("context_len", C.c_size_t)]


class _Sizes(C.Structure):
    _fields_ = [(k, C.c_size_t) for k in ("input_share_leader", "input_share_helper", "public_share", "prep_share",
                                          "prep_msg", "prep_state", "out_share", "agg_share")]


class _Prio3:
    KIND = 0

    def __init__(self, numShares, context=b"", **params):
        self._ctx = bytes(context)
        self._cfg = _Config(kind=self.KIND, num_shares=numShares, context=self._ctx, context_len=len(self._ctx),
                            **params)
        self.shares = numShares
        z = _Sizes()
        rc = lib().cb200_prio3_get_sizes(C.byref(self._cfg), C.byref(z))
        if rc:
            raise ValueError(lib().cb200_last_error().decode())
        self._z = {k: getattr(z, k) for k, _ in _Sizes._fields_}
        self.p = P64 if self.KIND <= 2 else P128
        self.elt = 8 if self.KIND <= 2 else 16

    def Params(self):
        return dict(self._z)

    # ---------------------------------------------------------------- batches
    def _rows(self, x, width, n, what):
        if width == 0:
            return None
        x = _prep(x, width, ValueError(f"{what}: expected (n, {width}) uint8 rows"))
        if x.shape[0] != n:
            raise ValueError(f"{what}: expected {n} rows")
        return x

    def PrepInitBatch(self, verifyKey, aggID, nonces, publicShares, inputShares):
        """(prep_states, prep_shares, status) of n reports as aggregator aggID"""
        z = self._z
        if len(verifyKey) != 32:
            raise ValueError("verify key must be 32 bytes")
        n = len(nonces)
        nonces = self._rows(nonces, 16, n, "nonces")
        pub = self._rows(publicShares, z["public_share"], n, "public shares")
        ins = self._rows(inputShares, z["input_share_helper" if aggID else "input_share_leader"], n, "input shares")
        states, shares, status = _new(nonces, (n, z["prep_state"])), _new(nonces, (n, z["prep_share"])), \
            _new(nonces, (n,))
        check(lib().cb200_prio3_prep_init(C.byref(self._cfg), bytes(verifyKey), aggID, _ptr(nonces),
                                          _ptr(pub) if pub is not None else None, _ptr(ins), _ptr(states),
                                          _ptr(shares), _ptr(status), n))
        return states, shares, status

    def PrepSharesToPrepBatch(self, prepShares):
        """prepShares: (n, shares * prep_share) rows, the aggregators' prep shares of each report in order ->
        (prep_msgs, status)"""
        z = self._z
        n = len(prepShares)
        rows = self._rows(prepShares, self.shares * z["prep_share"], n, "prep shares")
        msgs, status = _new(rows, (n, z["prep_msg"])), _new(rows, (n,))
        check(lib().cb200_prio3_prep_shares_to_prep(C.byref(self._cfg), _ptr(rows),
                                                    _ptr(msgs) if z["prep_msg"] else None, _ptr(status), n))
        return msgs, status

    def PrepNextBatch(self, prepStates, prepMsgs):
        """(out_shares, status)"""
        z = self._z
        n = len(prepStates)
        states = self._rows(prepStates, z["prep_state"], n, "prep states")
        msgs = self._rows(prepMsgs, z["prep_msg"], n, "prep messages")
        out, status = _new(states, (n, z["out_share"])), _new(states, (n,))
        check(lib().cb200_prio3_prep_next(C.byref(self._cfg), _ptr(states), _ptr(msgs) if msgs is not None else None,
                                          _ptr(out), _ptr(status), n))
        return out, status

    def AggregateBatch(self, outShares, status=None):
        """the agg share (bytes, or a CUDA tensor for CUDA rows) of the rows whose status byte is 0"""
        z = self._z
        n = len(outShares)
        rows = self._rows(outShares, z["out_share"], n, "out shares")
        if status is not None and not _is_torch(status):
            status = np.ascontiguousarray(status, dtype=np.uint8)
        agg = _new(rows, (z["agg_share"],))
        check(lib().cb200_prio3_aggregate(C.byref(self._cfg), _ptr(rows), _ptr(status) if status is not None else None,
                                          _ptr(agg), n))
        return agg if _is_torch(agg) else agg.tobytes()

    # ---------------------------------------------------------------- one report
    def PrepInit(self, verifyKey, nonce, aggID, publicShare, inputShare):
        """(prep_state, prep_share) as bytes"""
        pub = np.frombuffer(bytes(publicShare), np.uint8).reshape(1, -1) if self._z["public_share"] else None
        st, sh, status = self.PrepInitBatch(verifyKey, aggID, np.frombuffer(bytes(nonce), np.uint8).reshape(1, -1), pub,
                                            np.frombuffer(bytes(inputShare), np.uint8).reshape(1, -1))
        _raise(int(status[0]))
        return st[0].tobytes(), sh[0].tobytes()

    def PrepSharesToPrep(self, prepShares):
        if len(prepShares) != self.shares:
            raise ValueError("invalid prep shares length (ErrPrepShareSize)")
        msgs, status = self.PrepSharesToPrepBatch(np.frombuffer(b"".join(prepShares), np.uint8).reshape(1, -1))
        _raise(int(status[0]))
        return msgs[0].tobytes()

    def PrepNext(self, prepState, prepMsg):
        msgs = np.frombuffer(bytes(prepMsg), np.uint8).reshape(1, -1) if self._z["prep_msg"] else None
        out, status = self.PrepNextBatch(np.frombuffer(bytes(prepState), np.uint8).reshape(1, -1), msgs)
        _raise(int(status[0]))
        return out[0].tobytes()

    def AggregateInit(self):
        return bytes(self._z["agg_share"])

    def _elts(self, b):
        return [int.from_bytes(b[i:i + self.elt], "little") for i in range(0, len(b), self.elt)]

    def AggregateUpdate(self, aggShare, outShare):
        """aggShare + outShare, as bytes"""
        return self._merge([aggShare, outShare])

    def _merge(self, shares):
        acc = [0] * (self._z["agg_share"] // self.elt)
        for s in shares:
            acc = [(a + b) % self.p for a, b in zip(acc, self._elts(bytes(s)))]
        return b"".join(a.to_bytes(self.elt, "little") for a in acc)

    def Unshard(self, aggShares, numMeas):
        """the aggregate result: an int (Count, Sum) or a list of ints"""
        if len(aggShares) != self.shares:
            raise ValueError("invalid aggregate shares length (ErrAggShareSize)")
        out = self._elts(self._merge(aggShares))
        if any(x >> 64 for x in out):  # GetUint64 of a Field128 element
            raise ValueError("number of bits is not enough to represent the number")
        if self.KIND == 2:
            hi_max = numMeas * self._cfg.max_measurement
            if hi_max >= P64:
                raise ValueError("sum aggregate bound is not representable in Fp64")
        return out[0] if self.KIND <= 2 else out


class Count(_Prio3):
    KIND = 1

    def __init__(self, numShares, context=b""):
        super().__init__(numShares, context)


class Sum(_Prio3):
    KIND = 2

    def __init__(self, numShares, maxMeasurement, context=b""):
        super().__init__(numShares, context, max_measurement=maxMeasurement)


class SumVec(_Prio3):
    KIND = 3

    def __init__(self, numShares, length, bits, chunkLength, context=b""):
        super().__init__(numShares, context, length=length, bits=bits, chunk_length=chunkLength)


class Histogram(_Prio3):
    KIND = 4

    def __init__(self, numShares, length, chunkLength, context=b""):
        super().__init__(numShares, context, length=length, chunk_length=chunkLength)


class MultiHotCountVec(_Prio3):
    KIND = 5

    def __init__(self, numShares, length, maxWeight, chunkLength, context=b""):
        super().__init__(numShares, context, length=length, max_weight=maxWeight, chunk_length=chunkLength)
