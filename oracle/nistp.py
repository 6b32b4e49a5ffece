"""oracle.nistp -- TEST INFRASTRUCTURE ONLY.

ctypes view of ``oracle/liboracle_nistp.so``, the plain-C restatement of HPKE's DHKEM(P-384, HKDF-SHA384) and
DHKEM(P-521, HKDF-SHA512) (``oracle/nistp.c``) with its own textbook curve arithmetic, SHA-384 and SHA-512.  Every
call takes the curve as ``bits`` (384 or 521).  It is built on its own with gcc.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "nistp.c")
_LIB_PATH = os.path.join(_HERE, "liboracle_nistp.so")

KEM_ID = {384: 0x11, 521: 0x12}
NSK = {384: 48, 521: 66}
NPK = {384: 97, 521: 133}
NSS = {384: 48, 521: 64}


def build(force: bool = False) -> str:
    deps = [_SRC, os.path.join(_HERE, "oracle.h")]
    stale = not os.path.exists(_LIB_PATH) or any(os.path.getmtime(d) > os.path.getmtime(_LIB_PATH) for d in deps)
    if force or stale:
        subprocess.run([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-Wall", "-Wextra", "-std=c11", "-shared", "-o",
                        _LIB_PATH, _SRC], check=True, capture_output=True)
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


def scalar_ok(bits: int, sk: bytes) -> bool:
    """crypto/ecdh NewPrivateKey: 0 < k < n."""
    return len(sk) == NSK[bits] and bool(lib().orc_nistp_scalar_ok(bits, _buf(sk)))


def point_ok(bits: int, pk: bytes) -> bool:
    """crypto/ecdh NewPublicKey: 0x04 || X || Y with X, Y < p on the curve."""
    return len(pk) == NPK[bits] and bool(lib().orc_nistp_point_ok(bits, _buf(pk)))


def ecdh(bits: int, sk: bytes, pt: bytes | None = None):
    """(out, status): KeyGen (pt None: 0x04 || X || Y) or Shared (X); status bit 0 = bad point, bit 1 = bad scalar."""
    out = (C.c_uint8 * (NSK[bits] if pt is not None else NPK[bits]))()
    st = lib().orc_nistp(bits, out, _buf(sk), _opt(pt))
    return bytes(out), st


def sha384(m: bytes) -> bytes:
    out = (C.c_uint8 * 48)()
    lib().orc_sha384(out, _buf(m), C.c_size_t(len(m)))
    return bytes(out)


def keygen(bits: int, seed: bytes):
    """(pk, sk, ctr): DeriveKeyPair and the candidate counter that gave the key."""
    pk, sk = (C.c_uint8 * NPK[bits])(), (C.c_uint8 * NSK[bits])()
    ctr = lib().orc_nistp_derive(bits, pk, sk, _buf(seed))
    return bytes(pk), bytes(sk), ctr


def encaps(bits: int, pkR: bytes, seed: bytes, skS: bytes | None = None):
    """(enc, ss, status): Encap, or AuthEncap with skS; status bit 0 = invalid pkR, bit 1 = invalid skS (ss zero)."""
    enc, ss = (C.c_uint8 * NPK[bits])(), (C.c_uint8 * NSS[bits])()
    st = lib().orc_nistp_encaps(bits, enc, ss, _buf(pkR), _opt(skS), _buf(seed))
    return bytes(enc), bytes(ss), st


def decaps(bits: int, skR: bytes, enc: bytes, pkS: bytes | None = None):
    """(ss, status): Decap, or AuthDecap with pkS; status bit 0 = invalid enc / pkS, bit 1 = invalid skR."""
    ss = (C.c_uint8 * NSS[bits])()
    st = lib().orc_nistp_decaps(bits, ss, _buf(skR), _buf(enc), _opt(pkS))
    return bytes(ss), st
