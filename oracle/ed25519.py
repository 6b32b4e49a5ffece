"""oracle.ed25519 -- TEST INFRASTRUCTURE ONLY.

ctypes view of ``oracle/liboracle_ed25519.so``, the plain-C restatement of sign/ed25519 (pure Ed25519) and of
sign/eddilithium2 (``oracle/ed25519.c``).  It is built on its own with gcc and links against ``liboracle.so``
(``oracle.build()``) for SHAKE256 and round-3 Dilithium2.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "ed25519.c")
_LIB_PATH = os.path.join(_HERE, "liboracle_ed25519.so")


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
        _lib.orc_ed25519_verify.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
        _lib.orc_eddilithium2_verify.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
        _lib.orc_ed25519_sign.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
        _lib.orc_eddilithium2_sign.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
        _lib.orc_sha512.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    return _lib


def _buf(b) -> C.Array:
    return (C.c_uint8 * max(1, len(b))).from_buffer_copy(bytes(b) or b"\0")


def sha512(data: bytes) -> bytes:
    out = (C.c_uint8 * 64)()
    lib().orc_sha512(out, _buf(data), len(data))
    return bytes(out)


def ed25519_keygen(seed: bytes):
    """(pk 32, sk 64 = seed || pk): NewKeyFromSeed."""
    pk, sk = (C.c_uint8 * 32)(), (C.c_uint8 * 64)()
    lib().orc_ed25519_keygen(pk, sk, _buf(seed))
    return bytes(pk), bytes(sk)


def ed25519_sign(sk: bytes, msg: bytes) -> bytes:
    """Sign with the public half of sk as given."""
    sig = (C.c_uint8 * 64)()
    lib().orc_ed25519_sign(sig, _buf(sk), _buf(msg), len(msg))
    return bytes(sig)


def ed25519_verify(pk: bytes, msg: bytes, sig: bytes) -> bool:
    return bool(lib().orc_ed25519_verify(_buf(pk), _buf(msg), len(msg), _buf(sig), len(sig)))


def eddilithium2_keygen(seed: bytes):
    """(pk 1344, sk 2560)."""
    pk, sk = (C.c_uint8 * 1344)(), (C.c_uint8 * 2560)()
    lib().orc_eddilithium2_keygen(pk, sk, _buf(seed))
    return bytes(pk), bytes(sk)


def eddilithium2_sign(sk: bytes, msg: bytes) -> bytes:
    sig = (C.c_uint8 * 2484)()
    lib().orc_eddilithium2_sign(sig, _buf(sk), _buf(msg), len(msg))
    return bytes(sig)


def eddilithium2_verify(pk: bytes, msg: bytes, sig: bytes) -> bool:
    return bool(lib().orc_eddilithium2_verify(_buf(pk), _buf(msg), len(msg), _buf(sig), len(sig)))
