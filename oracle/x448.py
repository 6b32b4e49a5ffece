"""oracle.x448 -- TEST INFRASTRUCTURE ONLY.

ctypes view of ``oracle/liboracle_x448.so``, the plain-C restatement of dh/x448 and of the kem/hybrid schemes over
X448 (``oracle/x448.c``).  It is built on its own with gcc and links against ``liboracle.so`` (``oracle.build()``)
for SHAKE256 and the round-3 Kyber KEM.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "x448.c")
_LIB_PATH = os.path.join(_HERE, "liboracle_x448.so")

# scheme name -> K of its round-3 Kyber half (kem/hybrid/hybrid.go:83-93)
HYBRID_K = {"Kyber768-X448": 3, "Kyber1024-X448": 4}


def build(force: bool = False) -> str:
    base = oracle.build()
    deps = [_SRC, os.path.join(_HERE, "oracle.h"), base]
    stale = not os.path.exists(_LIB_PATH) or any(os.path.getmtime(d) > os.path.getmtime(_LIB_PATH) for d in deps)
    if force or stale:
        subprocess.run([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-Wall", "-Wextra", "-std=c11", "-shared", "-o",
                        _LIB_PATH, _SRC, "-L" + _HERE, "-l:liboracle.so", "-Wl,-rpath,$ORIGIN"],
                       check=True, capture_output=True)
    return _LIB_PATH


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_LIB_PATH)
    return _lib


def _buf(b) -> C.Array:
    return (C.c_uint8 * len(b)).from_buffer_copy(bytes(b))


def x448(scalar: bytes, point: bytes | None = None):
    """(out, ok): dh/x448 KeyGen (point None) or Shared; ok False for the low-order points 0, 1, p - 1."""
    out = (C.c_uint8 * 56)()
    ok = lib().orc_x448(out, _buf(scalar), _buf(point) if point is not None else None)
    return bytes(out), bool(ok)


def hybrid_sizes(name: str):
    """(pk, sk, ct) sizes: the 56-byte X448 half in front of the round-3 Kyber one."""
    eksz, dksz, ctsz = oracle.mlkem_sizes(HYBRID_K[name])
    return eksz + 56, dksz + 56, ctsz + 56


def hybrid_seed_sizes(name: str):
    """(shared secret, encapsulation seed) sizes: 56 + 32 and max(56, 32)."""
    if name not in HYBRID_K:
        raise KeyError(name)
    return 88, 56


def hybrid_keygen(name: str, seed64: bytes):
    pksz, sksz, _ = hybrid_sizes(name)
    pk, sk = (C.c_uint8 * pksz)(), (C.c_uint8 * sksz)()
    lib().orc_x448_hybrid_keygen(HYBRID_K[name], pk, sk, _buf(seed64))
    return bytes(pk), bytes(sk)


def hybrid_encaps(name: str, pk: bytes, seed56: bytes):
    """(ct, ss, rc): rc 1 = kem.ErrPubKey."""
    _, _, ctsz = hybrid_sizes(name)
    ct, ss = (C.c_uint8 * ctsz)(), (C.c_uint8 * 88)()
    rc = lib().orc_x448_hybrid_encaps(HYBRID_K[name], ct, ss, _buf(pk), _buf(seed56))
    return bytes(ct), bytes(ss), rc


def hybrid_decaps(name: str, sk: bytes, ct: bytes):
    """(ss, rc): rc 1 = kem.ErrPubKey (low-order X448 share)."""
    ss = (C.c_uint8 * 88)()
    rc = lib().orc_x448_hybrid_decaps(HYBRID_K[name], ss, _buf(sk), _buf(ct))
    return bytes(ss), rc
