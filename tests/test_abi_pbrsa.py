"""CPU-only: the partially blind RSA entry points are exported and listed; every argument error is CB200_ERR_ARG with
a message before the device is touched (keys outside the served range, primes not = 3 mod 4, qinv >= p, null pointers,
host offsets that decrease or span 2^31 bytes); cb200_pbrsa_check_key accepts the safe-prime fixture keys and refuses
keys whose primes are not safe; the Python constructors map these to the reference's errors; and with a good key the
entry points fail loudly without a device."""
import ctypes as C

import numpy as np
import pytest

import brsa_model as bm
import pbrsa_model as pm

NAMES = ("cb200_pbrsa_check_key", "cb200_pbrsa_blind_sign", "cb200_pbrsa_verify")
ERR_ARG, ERR_NOT_INIT = -1, -2


def _be(x):
    return x.to_bytes((x.bit_length() + 7) // 8 or 1, "big")


@pytest.fixture(scope="module")
def L():
    from circl_b200 import _ffi
    return _ffi.lib()


def _sign(L, n, p, q, qinv, count=1, meta_off=None, nulls=()):
    z = np.zeros(8192, np.uint8)
    off = np.zeros(count + 1, np.uint64) if meta_off is None else np.asarray(meta_off, np.uint64)
    key = [_be(n), _be(p), _be(q), _be(qinv)]
    bufs = [z.ctypes.data, z.ctypes.data, off.ctypes.data, z.ctypes.data, z.ctypes.data]
    args = []
    for i, f in enumerate(key):
        args += [None if i in nulls else f, len(f)]
    bufs = [None if 4 + i in nulls else b for i, b in enumerate(bufs)]
    return L.cb200_pbrsa_blind_sign(*args, *bufs, count)


def _verify(L, n, count=1, msg_off=None, meta_off=None, nulls=()):
    z = np.zeros(8192, np.uint8)
    mo = np.zeros(count + 1, np.uint64) if msg_off is None else np.asarray(msg_off, np.uint64)
    do = np.zeros(count + 1, np.uint64) if meta_off is None else np.asarray(meta_off, np.uint64)
    bufs = [z.ctypes.data, mo.ctypes.data, z.ctypes.data, do.ctypes.data, z.ctypes.data, z.ctypes.data]
    bufs = [None if 1 + i in nulls else b for i, b in enumerate(bufs)]
    nb = _be(n)
    return L.cb200_pbrsa_verify(None if 0 in nulls else nb, len(nb), *bufs, count)


def _good(k):
    return k.n, k.p, k.q, pow(k.q, -1, k.p)


def test_exports_and_symbols():
    from circl_b200 import _ffi
    raw = C.CDLL(_ffi.lib()._name)
    for name in NAMES:
        assert hasattr(raw, name) and name in _ffi.SYMBOLS, name


def test_argument_errors(L):
    k = pm.keys()["strong2048"]
    n, p, q, qinv = _good(k)
    small = bm.Key(p * 3, 65537, 0, p, 3)  # 1026 bits
    cases = {
        "1026-bit modulus": (small.n, p, 3, 1),
        "8192-bit modulus": (n ** 4, p, q, qinv),
        "p q != N": (n, p + 4, q, qinv),
        "qinv = p": (n, p, q, p),
        "qinv > p": (n, p, q, p + 1),
    }
    for name, f in cases.items():
        assert _sign(L, *f) == ERR_ARG, name
        assert L.cb200_last_error(), name
    # primes = 1 mod 4 (so p' would be even): N = p q with p = 1 mod 4
    u = bm.all_keys()["rsa3072"]
    p1 = next(x for x in (u.p, u.q) if x % 4 == 1)
    assert _sign(L, u.n, p1, u.n // p1, pow(u.n // p1, -1, p1)) == ERR_ARG
    assert b"3 mod 4" in L.cb200_last_error()
    assert L.cb200_pbrsa_check_key(_be(u.n), len(_be(u.n)), _be(p1), len(_be(p1)), _be(u.n // p1),
                                   len(_be(u.n // p1))) == ERR_ARG
    # a larger prime over 2048 bits
    big_p = (1 << 2050) + 3  # the range is checked before any primality
    nb = big_p * 7
    assert 2048 <= nb.bit_length() <= 4096
    assert _sign(L, nb, big_p, 7, 1) == ERR_ARG and b"2051 bits" in L.cb200_last_error()
    for i in range(9):  # N, p, q, qinv, blinded, meta, meta_off, sig, status
        assert _sign(L, n, p, q, qinv, nulls=(i,)) == ERR_ARG, i
        assert b"null" in L.cb200_last_error()
    assert _sign(L, n, p, q, qinv, count=2, meta_off=[0, 5, 4]) == ERR_ARG
    assert b"decreases" in L.cb200_last_error()
    assert _sign(L, n, p, q, qinv, count=2, meta_off=[0, 1, 1 << 31]) == ERR_ARG
    assert b"2^31" in L.cb200_last_error()
    # Verify
    assert _verify(L, small.n) == ERR_ARG
    assert _verify(L, n ** 4) == ERR_ARG
    for i in range(7):  # N, msgs, msg_off, meta, meta_off, sigs, status
        assert _verify(L, n, nulls=(i,)) == ERR_ARG, i
    assert _verify(L, n, count=2, msg_off=[0, 3, 2]) == ERR_ARG
    assert _verify(L, n, count=2, meta_off=[0, 3, 2]) == ERR_ARG
    assert _verify(L, n, count=1, msg_off=[0, 1 << 30], meta_off=[0, 1 << 30]) == ERR_ARG
    assert b"2^31" in L.cb200_last_error()
    assert _verify(L, n, count=1, msg_off=[0, 1 << 31]) == ERR_ARG


def test_check_key(L):
    for name, k in pm.keys().items():
        f = [_be(x) for x in (k.n, k.p, k.q)]
        assert L.cb200_pbrsa_check_key(f[0], len(f[0]), f[1], len(f[1]), f[2], len(f[2])) == 0, name
    weak = bm.all_keys()["rsa2048u"]  # primes = 3 mod 4 whose halves are composite
    assert weak.p % 4 == 3 and weak.q % 4 == 3
    f = [_be(x) for x in (weak.n, weak.p, weak.q)]
    assert L.cb200_pbrsa_check_key(f[0], len(f[0]), f[1], len(f[1]), f[2], len(f[2])) == ERR_ARG
    assert b"safe prime" in L.cb200_last_error()
    s = pm.keys()["strong2048"]
    f = [_be(x) for x in (s.n, s.p, s.q)]
    assert L.cb200_pbrsa_check_key(f[0], len(f[0]), f[1], len(f[1]), f[2][:-1], len(f[2]) - 1) == ERR_ARG
    assert L.cb200_pbrsa_check_key(None, 0, f[1], len(f[1]), f[2], len(f[2])) == ERR_ARG


def test_python_constructors():
    from circl_b200 import blindrsa, partiallyblindrsa as pb
    k = pm.keys()["strong2048"]
    sk = blindrsa.PrivateKey(k.n, k.e, k.d, [k.p, k.q])
    s = pb.NewSigner(sk, pb.SHA384)  # a good key constructs without a device
    assert s.kLen == 256
    pb.NewVerifier(sk.PublicKey, pb.SHA384)
    with pytest.raises(ValueError, match="SHA384"):
        pb.NewSigner(sk, "SHA256")
    with pytest.raises(ValueError, match="SHA384"):
        pb.NewVerifier(sk.PublicKey, "SHA512")
    w = bm.all_keys()["rsa2048u"]
    with pytest.raises(pb.ErrInvalidPrivateKey, match="safe prime"):
        pb.NewSigner(blindrsa.PrivateKey(w.n, w.e, w.d, [w.p, w.q]))
    with pytest.raises(pb.ErrInvalidPrivateKey, match="p q = N"):
        pb.NewSigner(blindrsa.PrivateKey(k.n, k.e, k.d, [k.p + 4, k.q]))
    with pytest.raises(pb.ErrInvalidPrivateKey):
        pb.NewSigner(blindrsa.PrivateKey(k.n, k.e, k.d, [k.p, k.q, 3]))
    with pytest.raises(pb.ErrInvalidPublicKey):
        pb.NewVerifier(blindrsa.PublicKey(k.p, 3))
    with pytest.raises(pb.ErrUnexpectedSize):
        s.BlindSign(bytes(255), b"")
    assert pb.ErrVerification is blindrsa.ErrVerification and pb.ErrInternal is blindrsa.ErrInternal


def test_entry_points_without_a_device(L):
    for k in pm.keys().values():
        assert _sign(L, *_good(k)) == ERR_NOT_INIT
        assert _verify(L, k.n) == ERR_NOT_INIT
