"""oracle.p256 -- TEST INFRASTRUCTURE ONLY.

ctypes view of ``oracle/liboracle_p256.so``, the plain-C restatement of HPKE's DHKEM(P-256, HKDF-SHA256)
(``oracle/p256.c``) with its own textbook P-256 arithmetic.  It is built on its own with gcc and links against
``liboracle_hpke.so`` for SHA-256.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

from oracle import hpke as oracle_hpke

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "p256.c")
_LIB_PATH = os.path.join(_HERE, "liboracle_p256.so")

KEM_ID = 0x10
NSK, NPK, NSS = 32, 65, 32


def build(force: bool = False) -> str:
    base = oracle_hpke.build()
    deps = [_SRC, os.path.join(_HERE, "oracle.h"), base]
    stale = not os.path.exists(_LIB_PATH) or any(os.path.getmtime(d) > os.path.getmtime(_LIB_PATH) for d in deps)
    if force or stale:
        subprocess.run([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-Wall", "-Wextra", "-std=c11", "-shared", "-o",
                        _LIB_PATH, _SRC, "-L" + _HERE, "-l:liboracle_hpke.so", "-Wl,-rpath,$ORIGIN"],
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
    return (C.c_uint8 * max(1, len(b))).from_buffer_copy(bytes(b) or b"\0")


def _opt(b):
    return _buf(b) if b is not None else None


def scalar_ok(sk: bytes) -> bool:
    """crypto/ecdh NewPrivateKey: 0 < k < n."""
    return bool(lib().orc_p256_scalar_ok(_buf(sk)))


def point_ok(pk: bytes) -> bool:
    """crypto/ecdh NewPublicKey: 0x04 || X || Y with X, Y < p on the curve."""
    return len(pk) == NPK and bool(lib().orc_p256_point_ok(_buf(pk)))


def ecdh(sk: bytes, pt: bytes | None = None):
    """(out, status): KeyGen (pt None: 0x04 || X || Y) or Shared (X); status bit 0 = bad point, bit 1 = bad scalar."""
    out = (C.c_uint8 * (32 if pt is not None else 65))()
    st = lib().orc_p256(out, _buf(sk), _opt(pt))
    return bytes(out), st


def keygen(seed: bytes):
    """(pk, sk, ctr): DeriveKeyPair and the candidate counter that gave the key."""
    pk, sk = (C.c_uint8 * NPK)(), (C.c_uint8 * NSK)()
    ctr = lib().orc_p256_derive(pk, sk, _buf(seed))
    return bytes(pk), bytes(sk), ctr


def encaps(pkR: bytes, seed: bytes, skS: bytes | None = None):
    """(enc, ss, status): Encap, or AuthEncap with skS; status bit 0 = invalid pkR, bit 1 = invalid skS (ss zero)."""
    enc, ss = (C.c_uint8 * NPK)(), (C.c_uint8 * NSS)()
    st = lib().orc_p256_encaps(enc, ss, _buf(pkR), _opt(skS), _buf(seed))
    return bytes(enc), bytes(ss), st


def decaps(skR: bytes, enc: bytes, pkS: bytes | None = None):
    """(ss, status): Decap, or AuthDecap with pkS; status bit 0 = invalid enc / pkS, bit 1 = invalid skR."""
    ss = (C.c_uint8 * NSS)()
    st = lib().orc_p256_decaps(ss, _buf(skR), _buf(enc), _opt(pkS))
    return bytes(ss), st
