"""oracle.frodo -- TEST INFRASTRUCTURE ONLY.

ctypes view of ``oracle/liboracle_frodo.so``, the plain-C restatement of FrodoKEM-640-SHAKE (``oracle/frodo.c``).  It is
built on its own with gcc and links against ``liboracle.so`` (``oracle.build()``) for SHAKE128.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "frodo.c")
_LIB_PATH = os.path.join(_HERE, "liboracle_frodo.so")

PK, SK, CT, SS, SEED, ESEED = 9616, 19888, 9720, 16, 48, 16


def build(force: bool = False) -> str:
    base = oracle.build()
    deps = [_SRC, os.path.join(_HERE, "oracle.h"), base]
    stale = not os.path.exists(_LIB_PATH) or any(os.path.getmtime(d) > os.path.getmtime(_LIB_PATH) for d in deps)
    if force or stale:
        subprocess.run([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-Wall", "-Wextra", "-std=c11", "-shared", "-o",
                        _LIB_PATH, _SRC, "-L" + _HERE, "-l:liboracle.so", "-lpthread", "-Wl,-rpath,$ORIGIN"],
                       check=True, capture_output=True)
    return _LIB_PATH


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_LIB_PATH)
        _lib.orc_frodo_sample.restype = C.c_uint16
        _lib.orc_frodo_sample.argtypes = [C.c_uint16]
        _lib.orc_frodo_batch.argtypes = [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_size_t, C.c_int]
    return _lib


def _buf(b) -> C.Array:
    return (C.c_uint8 * len(b)).from_buffer_copy(bytes(b))


def keygen(seed: bytes):
    """(pk, sk): DeriveKeyPair of a 48-byte seed."""
    pk, sk = (C.c_uint8 * PK)(), (C.c_uint8 * SK)()
    lib().orc_frodo_keygen(pk, sk, _buf(seed))
    return bytes(pk), bytes(sk)


def encaps(pk: bytes, seed: bytes):
    """(ct, ss): EncapsulateDeterministically with a 16-byte seed."""
    ct, ss = (C.c_uint8 * CT)(), (C.c_uint8 * SS)()
    lib().orc_frodo_encaps(ct, ss, _buf(pk), _buf(seed))
    return bytes(ct), bytes(ss)


def decaps(sk: bytes, ct: bytes) -> bytes:
    ss = (C.c_uint8 * SS)()
    lib().orc_frodo_decaps(ss, _buf(sk), _buf(ct))
    return bytes(ss)


def sample(r: int) -> int:
    return lib().orc_frodo_sample(r)


def pack(v) -> bytes:
    v = np.ascontiguousarray(v, dtype=np.uint16)
    out = (C.c_uint8 * (15 * v.size // 8))()
    lib().orc_frodo_pack(out, v.ctypes.data_as(C.c_void_p), C.c_size_t(v.size))
    return bytes(out)


def unpack(b: bytes):
    out = np.zeros(8 * len(b) // 15, dtype=np.uint16)
    lib().orc_frodo_unpack(out.ctypes.data_as(C.c_void_p), _buf(b), C.c_size_t(len(b)))
    return out


def _rows(x, w):
    x = np.ascontiguousarray(x, dtype=np.uint8)
    return x.reshape(-1, w)


def keygen_batch(seeds, nthreads: int = 1):
    s = _rows(seeds, SEED)
    n = s.shape[0]
    pk, sk = np.empty((n, PK), np.uint8), np.empty((n, SK), np.uint8)
    lib().orc_frodo_batch(0, None, 0, s.ctypes.data, pk.ctypes.data, sk.ctypes.data, n, nthreads)
    return pk, sk


def encaps_batch(pks, seeds, nthreads: int = 1):
    """pks: (n, 9616), or one (9616,) row shared by the batch."""
    s = _rows(seeds, ESEED)
    n = s.shape[0]
    k = np.ascontiguousarray(pks, dtype=np.uint8)
    stride = 0 if k.ndim == 1 else PK
    ct, ss = np.empty((n, CT), np.uint8), np.empty((n, SS), np.uint8)
    lib().orc_frodo_batch(1, k.ctypes.data, stride, s.ctypes.data, ct.ctypes.data, ss.ctypes.data, n, nthreads)
    return ct, ss


def decaps_batch(sks, cts, nthreads: int = 1):
    """sks: (n, 19888), or one (19888,) row shared by the batch."""
    c = _rows(cts, CT)
    n = c.shape[0]
    k = np.ascontiguousarray(sks, dtype=np.uint8)
    stride = 0 if k.ndim == 1 else SK
    ss = np.empty((n, SS), np.uint8)
    lib().orc_frodo_batch(2, k.ctypes.data, stride, c.ctypes.data, None, ss.ctypes.data, n, nthreads)
    return ss
