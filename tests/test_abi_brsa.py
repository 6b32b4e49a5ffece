"""CPU-only: the RSA blind-signature entry points are exported and listed, refuse every key outside the served range
with CB200_ERR_ARG and a message (multi-prime, p q != N, even e, 1024- and 8192-bit moduli), and fail loudly without a
device on a good key."""
import ctypes as C

import numpy as np
import pytest

import brsa_model as bm

NAMES = ("cb200_brsa_blind_sign", "cb200_brsa_verify", "cb200_brsa_modulus_bytes")


def _be(x):
    return x.to_bytes((x.bit_length() + 7) // 8 or 1, "big")


def test_exports_and_symbols():
    from circl_b200 import _ffi
    L = C.CDLL(_ffi.lib()._name)
    for name in NAMES:
        assert hasattr(L, name) and name in _ffi.SYMBOLS, name
    L = _ffi.lib()
    for name, k in bm.all_keys().items():
        n = _be(k.n)
        assert L.cb200_brsa_modulus_bytes(n, len(n)) == k.klen, name
        assert L.cb200_brsa_modulus_bytes(b"\0\0" + n, len(n) + 2) == k.klen
    assert L.cb200_brsa_modulus_bytes(b"\x01" + bytes(128), 129) == 0


def _sign(L, fields, n=1):
    z = np.zeros(4096, np.uint8)
    args = []
    for f in fields:
        args += [f, len(f)]
    return L.cb200_brsa_blind_sign(*args, z.ctypes.data, z.ctypes.data, z.ctypes.data, n)


def _verify(L, n_, e, variant=0):
    z = np.zeros(4096, np.uint8)
    off = np.zeros(2, np.uint64)
    return L.cb200_brsa_verify(variant, n_, len(n_), e, len(e), z.ctypes.data, off.ctypes.data, z.ctypes.data,
                               z.ctypes.data, 1)


def _fields(k, **over):
    dp, dq, qinv = k.crt()
    f = {**dict(n=k.n, e=k.e, p=k.p, q=k.q, dp=dp, dq=dq, qinv=qinv), **over}
    return [_be(f[x]) for x in ("n", "e", "p", "q", "dp", "dq", "qinv")]


def _small_key(bits, rng_seed, e=65537):
    import random
    rng = random.Random(rng_seed)

    def prime(b):
        while True:
            p = rng.getrandbits(b) | (3 << (b - 2)) | 1
            if (p - 1) % e and all(pow(a, p - 1, p) == 1 for a in (2, 3, 5, 7, 11, 13)):
                return p
    p, q = prime(bits // 2), prime(bits // 2)
    return bm.Key(p * q, e, pow(e, -1, (p - 1) * (q - 1)), p, q)


def test_bad_keys_are_argument_errors():
    from circl_b200 import _ffi
    L = _ffi.lib()
    k = bm.pem_key()
    bad = {
        "p q != N": _fields(k, p=k.p + 2),
        "multi-prime (p, q of a three-prime N)": _fields(k, n=k.n * 65537),
        "even e": _fields(k, e=65536),
        "e = 1": _fields(k, e=1),
        "e >= 2^32": _fields(k, e=2**32 + 1),
        "dp wider than the primes": _fields(k, dp=1 << 1100),
    }
    for name, f in bad.items():
        assert _sign(L, f) == -1, name
        assert L.cb200_last_error(), name
    k1024 = _small_key(1024, 1)
    assert _sign(L, _fields(k1024)) == -1
    assert b"1024 bits" in L.cb200_last_error()
    assert _verify(L, _be(k1024.n), _be(k1024.e)) == -1
    big = bm.Key(k.n * k.n * k.n * k.n, k.e, 0, k.p, k.q)  # 8192 bits
    assert _verify(L, _be(big.n), _be(big.e)) == -1
    assert _sign(L, _fields(big, n=big.n)) == -1
    assert _verify(L, _be(k.n), _be(65536)) == -1
    assert _verify(L, _be(k.n), _be(k.e), variant=4) == -1
    assert _verify(L, _be(k.n), _be(k.e), variant=-1) == -1


def test_larger_prime_over_2048_bits():
    """a two-prime modulus in range whose larger prime is over 2048 bits is refused with its own message"""
    import random
    from circl_b200 import _ffi, blindrsa
    rng = random.Random(2050)
    p, q = rng.getrandbits(2050) | (1 << 2049) | 1, rng.getrandbits(1950) | (1 << 1949) | 1
    k = bm.Key(p * q, 65537, 3, p, q)
    assert 2048 <= k.n.bit_length() <= 4096
    L = _ffi.lib()
    assert _sign(L, _fields(k, dp=3, dq=3, qinv=3)) == -1
    assert b"larger prime has 2050 bits" in L.cb200_last_error()
    blindrsa.NewVerifier(0, blindrsa.PublicKey(k.n, k.e))  # its public key is served
    with pytest.raises(blindrsa.ErrInvalidKey, match="2050 bits"):
        blindrsa.NewSigner(blindrsa.PrivateKey(k.n, k.e, 2**64 + 1, [p, q]))


def test_python_key_checks():
    from circl_b200 import blindrsa
    k = bm.pem_key()
    blindrsa.NewSigner(blindrsa.PrivateKey(k.n, k.e, k.d, [k.p, k.q]))  # a good key constructs without a device
    blindrsa.NewVerifier(3, blindrsa.PublicKey(k.n, k.e))
    with pytest.raises(blindrsa.ErrInvalidKey, match="p q = N"):
        blindrsa.NewSigner(blindrsa.PrivateKey(k.n, k.e, k.d, [k.p + 2, k.q]))
    with pytest.raises(blindrsa.ErrInvalidKey, match="exponent"):
        blindrsa.NewVerifier(0, blindrsa.PublicKey(k.n, 65536))
    with pytest.raises(blindrsa.ErrInvalidKey):
        blindrsa.NewSigner(blindrsa.PrivateKey(k.n * 3, k.e, k.d, [k.p, k.q, 3]))
    with pytest.raises(blindrsa.ErrInvalidVariant):
        blindrsa.NewVerifier(4, blindrsa.PublicKey(k.n, k.e))


def test_entry_points_without_a_device():
    from circl_b200 import _ffi
    L = _ffi.lib()
    for k in bm.all_keys().values():
        assert _sign(L, _fields(k)) == -2
        assert _verify(L, _be(k.n), _be(k.e)) == -2
