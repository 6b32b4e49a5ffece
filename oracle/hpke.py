"""oracle.hpke -- TEST INFRASTRUCTURE ONLY.

ctypes view of ``oracle/liboracle_hpke.so``, the plain-C restatement of HPKE's DHKEM(X25519, HKDF-SHA256) and
DHKEM(X448, HKDF-SHA512) (``oracle/hpke.c``).  It is built on its own with gcc and links against ``liboracle.so``
(X25519) and ``liboracle_x448.so`` (X448).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import oracle
from oracle import x448 as oracle_x448

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "hpke.c")
_LIB_PATH = os.path.join(_HERE, "liboracle_hpke.so")

# kem_id -> (N = key / enc / seed bytes, shared secret bytes)
SIZES = {0x20: (32, 32), 0x21: (56, 64)}


def build(force: bool = False) -> str:
    base = oracle.build()
    x448 = oracle_x448.build()
    deps = [_SRC, os.path.join(_HERE, "oracle.h"), base, x448]
    stale = not os.path.exists(_LIB_PATH) or any(os.path.getmtime(d) > os.path.getmtime(_LIB_PATH) for d in deps)
    if force or stale:
        subprocess.run([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-Wall", "-Wextra", "-std=c11", "-shared", "-o",
                        _LIB_PATH, _SRC, "-L" + _HERE, "-l:liboracle_x448.so", "-l:liboracle.so", "-Wl,-rpath,$ORIGIN"],
                       check=True, capture_output=True)
    return _LIB_PATH


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_LIB_PATH)
        _lib.orc_sha256.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
        _lib.orc_sha512.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    return _lib


def _buf(b) -> C.Array:
    return (C.c_uint8 * max(1, len(b))).from_buffer_copy(bytes(b) or b"\0")


def _opt(b):
    return _buf(b) if b is not None else None


def sha256(m: bytes) -> bytes:
    out = (C.c_uint8 * 32)()
    lib().orc_sha256(out, _buf(m), len(m))
    return bytes(out)


def sha512(m: bytes) -> bytes:
    out = (C.c_uint8 * 64)()
    lib().orc_sha512(out, _buf(m), len(m))
    return bytes(out)


def keygen(kem_id: int, seed: bytes):
    """(pk, sk): DeriveKeyPair."""
    n, _ = SIZES[kem_id]
    pk, sk = (C.c_uint8 * n)(), (C.c_uint8 * n)()
    assert lib().orc_hpke_keygen(kem_id, pk, sk, _buf(seed)) == 0
    return bytes(pk), bytes(sk)


def encaps(kem_id: int, pkR: bytes, seed: bytes, skS: bytes | None = None):
    """(enc, ss, rc): Encap, or AuthEncap with skS; rc 1 = hpke.ErrInvalidKEMSharedSecret (ss zero)."""
    n, nss = SIZES[kem_id]
    enc, ss = (C.c_uint8 * n)(), (C.c_uint8 * nss)()
    rc = lib().orc_hpke_encaps(kem_id, enc, ss, _buf(pkR), _opt(skS), _buf(seed))
    return bytes(enc), bytes(ss), rc


def decaps(kem_id: int, skR: bytes, enc: bytes, pkS: bytes | None = None):
    """(ss, rc): Decap, or AuthDecap with pkS."""
    _, nss = SIZES[kem_id]
    ss = (C.c_uint8 * nss)()
    rc = lib().orc_hpke_decaps(kem_id, ss, _buf(skR), _buf(enc), _opt(pkS))
    return bytes(ss), rc
