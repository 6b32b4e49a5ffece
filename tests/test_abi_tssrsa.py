"""CPU-only: the threshold RSA entry points are exported, listed in _ffi.SYMBOLS and declared in the header; every
argument outside the served range (modulus size, e, players, threshold, k, the share exponent's bound, null pointers)
is CB200_ERR_ARG with a message, without a device; and good arguments fail loudly without one."""
import ctypes as C
import math
import os

import numpy as np

import brsa_model as bm

NAMES = ("cb200_tssrsa_sign_share", "cb200_tssrsa_combine")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _be(x):
    return x.to_bytes((x.bit_length() + 7) // 8 or 1, "big")


def test_exports_and_symbols():
    from circl_b200 import _ffi
    L = C.CDLL(_ffi.lib()._name)
    header = open(os.path.join(ROOT, "include", "circl_b200.h")).read()
    for name in NAMES:
        assert hasattr(L, name) and name in _ffi.SYMBOLS and name + "(" in header, name


def _sign(L, n, players, E, buf=True):
    z = np.zeros(4096, np.uint8)
    p = z.ctypes.data if buf else None
    return L.cb200_tssrsa_sign_share(n, len(n), players, E, len(E), p, z.ctypes.data, 1)


def _combine(L, n, e, players, threshold, k, null=None):
    z = np.zeros(1 << 20, np.uint8)
    ptrs = [z.ctypes.data] * 5
    if null is not None:
        ptrs[null] = None
    return L.cb200_tssrsa_combine(n, len(n), e, len(e), players, threshold, k, *ptrs, 1)


def test_argument_errors():
    from circl_b200 import _ffi
    L = _ffi.lib()
    k = bm.all_keys()["rsa2048"]
    n, e = _be(k.n), _be(k.e)
    bound = k.n.bit_length() - 2 + (2 * math.factorial(3)).bit_length()
    small = bm.Key(k.p * 3, 3, 1, k.p, 3)
    cases_sign = [
        ("modulus under 2048 bits", (_be(small.n), 3, b"\x05")),
        ("modulus over 4096 bits", (_be(k.n ** 3), 3, b"\x05")),
        ("players 1", (n, 1, b"\x05")),
        ("players 65", (n, 65, b"\x05")),
        ("E over the bound", (n, 3, _be(1 << bound))),
    ]
    for what, args in cases_sign:
        assert _sign(L, *args) == -1, what
        assert L.cb200_last_error(), what
    assert b"bits; 2 Delta s_i has at most" in (_sign(L, n, 3, _be(1 << bound)) == -1 and L.cb200_last_error())
    assert _sign(L, n, 3, b"\x05", buf=False) == -1
    cases_comb = [
        ("modulus under 2048 bits", (_be(small.n), e, 3, 2, 2)),
        ("even e", (n, _be(65536), 3, 2, 2)),
        ("e = 1", (n, b"\x01", 3, 2, 2)),
        ("e >= 2^32", (n, _be(2**32 + 1), 3, 2, 2)),
        ("players 1", (n, e, 1, 1, 1)),
        ("players 65", (n, e, 65, 2, 2)),
        ("threshold 0", (n, e, 3, 0, 2)),
        ("threshold above players", (n, e, 3, 4, 4)),
        ("k below threshold", (n, e, 5, 3, 2)),
        ("k over 64", (n, e, 64, 2, 65)),
    ]
    for what, args in cases_comb:
        assert _combine(L, *args) == -1, what
        assert L.cb200_last_error(), what
    for i in range(5):
        assert _combine(L, n, e, 3, 2, 2, null=i) == -1
        assert b"null pointer" in L.cb200_last_error()


def test_entry_points_without_a_device():
    from circl_b200 import _ffi
    L = _ffi.lib()
    for k in bm.all_keys().values():
        n, e = _be(k.n), _be(k.e)
        assert _sign(L, n, 64, _be((1 << (k.n.bit_length() - 2)) * math.factorial(64))) == -2
        assert _combine(L, n, e, 64, 33, 64) == -2
