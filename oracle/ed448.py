"""oracle.ed448 -- TEST INFRASTRUCTURE ONLY.

ctypes view of ``oracle/liboracle_ed448.so``, the plain-C restatement of sign/ed448 (pure Ed448, with the isogeny
route of goldilocks CombinedMult and the reference's scalar arithmetic) and of sign/eddilithium3 (``oracle/ed448.c``).
It is built on its own with gcc and links against ``liboracle.so`` (``oracle.build()``) for SHAKE256 and round-3
Dilithium3.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "ed448.c")
_LIB_PATH = os.path.join(_HERE, "liboracle_ed448.so")


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
        _lib.orc_ed448_sign.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
        _lib.orc_ed448_verify.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p,
                                          C.c_size_t]
        _lib.orc_eddilithium3_sign.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
        _lib.orc_eddilithium3_verify.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    return _lib


def _buf(b) -> C.Array:
    return (C.c_uint8 * max(1, len(b))).from_buffer_copy(bytes(b) or b"\0")


def base_mult(k: int) -> bytes:
    """encode(ScalarBaseMult(k)) for k < l, through the twist."""
    out = (C.c_uint8 * 57)()
    lib().orc_ed448_base_mult(out, _buf(k.to_bytes(56, "little")))
    return bytes(out)


def ed448_keygen(seed: bytes):
    """(pk 57, sk 114 = seed || pk): NewKeyFromSeed."""
    pk, sk = (C.c_uint8 * 57)(), (C.c_uint8 * 114)()
    lib().orc_ed448_keygen(pk, sk, _buf(seed))
    return bytes(pk), bytes(sk)


def ed448_sign(sk: bytes, msg: bytes, ctx: bytes = b"") -> bytes:
    """Sign with the public half of sk as given; ValueError for a context over 255 bytes (the reference panics)."""
    sig = (C.c_uint8 * 114)()
    if lib().orc_ed448_sign(sig, _buf(sk), _buf(msg), len(msg), _buf(ctx), len(ctx)) != 0:
        raise ValueError("ed448: bad context length")
    return bytes(sig)


def ed448_verify(pk: bytes, msg: bytes, sig: bytes, ctx: bytes = b"") -> bool:
    return bool(lib().orc_ed448_verify(_buf(pk), _buf(msg), len(msg), _buf(sig), len(sig), _buf(ctx), len(ctx)))


def eddilithium3_keygen(seed: bytes):
    """(pk 2009, sk 4057)."""
    pk, sk = (C.c_uint8 * 2009)(), (C.c_uint8 * 4057)()
    lib().orc_eddilithium3_keygen(pk, sk, _buf(seed))
    return bytes(pk), bytes(sk)


def eddilithium3_sign(sk: bytes, msg: bytes) -> bytes:
    sig = (C.c_uint8 * 3407)()
    lib().orc_eddilithium3_sign(sig, _buf(sk), _buf(msg), len(msg))
    return bytes(sig)


def eddilithium3_verify(pk: bytes, msg: bytes, sig: bytes) -> bool:
    return bool(lib().orc_eddilithium3_verify(_buf(pk), _buf(msg), len(msg), _buf(sig), len(sig)))
