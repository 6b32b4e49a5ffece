"""Oracle pins for dh/x448 and the X448 hybrids: X448 against the reference's own RFC 7748 vectors
(dh/x448/key_test.go) and OpenSSL's X448; Kyber768-X448 / Kyber1024-X448 rebuilt from parts (OpenSSL X448,
SHAKE256 and the oracle's round-3 Kyber KEM), since the reference has no vectors for them."""
import hashlib
import os
import subprocess

import pytest
from cryptography.hazmat.primitives.asymmetric.x448 import X448PrivateKey, X448PublicKey

import oracle
from conftest import load_golden
from oracle import x448 as ox

P = 2**448 - 2**224 - 1
BASE = bytes([5] + [0] * 55)


def _le(x):
    return x.to_bytes(56, "little")


def _openssl(k, u):
    """OpenSSL's X448, or None where it refuses the all-zero result."""
    try:
        return X448PrivateKey.from_private_bytes(k).exchange(X448PublicKey.from_public_bytes(u))
    except ValueError:
        return None


@pytest.fixture(scope="module")
def xv():
    return load_golden("x448_vectors.json.gz")


def test_rfc7748_kat(xv):
    assert len(xv["rfc7748_kat"]) == 6
    for v in xv["rfc7748_kat"]:  # key_test.go:23-45
        out, _ = ox.x448(bytes.fromhex(v["scalar"]), bytes.fromhex(v["input"]))
        assert out.hex() == v["output"]


def test_rfc7748_iterated(xv):
    assert [v["times"] for v in xv["rfc7748_times"]] == [1, 1000]  # 10^6 skipped, as key_test.go:69 does
    for v in xv["rfc7748_times"]:  # key_test.go:53-79
        u = k = BASE
        for _ in range(v["times"]):
            r, _ = ox.x448(k, u)
            u, k = k, r
        assert k.hex() == v["key"]


def test_keygen_equals_shared_with_base_point():
    for i in range(64):
        k = hashlib.shake_256(b"x448-%d" % i).digest(56)
        assert ox.x448(k)[0] == ox.x448(k, BASE)[0]


def test_against_openssl_random_and_non_canonical():
    for i in range(200):
        k = hashlib.shake_256(b"k%d" % i).digest(56)
        u = hashlib.shake_256(b"u%d" % i).digest(56)
        out, ok = ox.x448(k, u)
        assert ok and out == _openssl(k, u), i
        assert ox.x448(k)[0] == X448PrivateKey.from_private_bytes(k).public_key().public_bytes_raw()
    # non-canonical u: p, p + 1 and 2^448 - 1 are taken as their residues 0, 1 and 2^224
    for u in (P, P + 1, 2**448 - 1):
        for i in range(8):
            k = hashlib.shake_256(b"n%d-%d" % (u % 7, i)).digest(56)
            out, ok = ox.x448(k, _le(u))
            want = _openssl(k, _le(u))
            if want is None:  # OpenSSL refuses an all-zero result: the oracle must reject it as well
                assert out == bytes(56) and not ok
            else:
                assert ok and out == want


def test_low_order_points():
    for u in (0, 1, P - 1, P, P + 1):  # curve.go:76-104, reduced mod p first (key.go:22-30)
        out, ok = ox.x448(hashlib.shake_256(b"lo").digest(56), _le(u))
        assert out == bytes(56) and not ok, u


def _hybrid_from_parts(name, k, seed64, eseed56):
    """hybrid.go:197-261 over xkem.go:112-178 with OpenSSL X448 and hashlib SHAKE256."""
    ex = hashlib.shake_256(seed64).digest(56 + 64)
    skx = hashlib.shake_256(ex[:56]).digest(56)
    pkx = X448PrivateKey.from_private_bytes(skx).public_key().public_bytes_raw()
    ek, dk = oracle.kyber_kem_keygen(k, ex[56:])
    pk, sk = pkx + ek, skx + dk
    ee = hashlib.shake_256(eseed56).digest(56 + 32)
    esk = hashlib.shake_256(ee[:56]).digest(56)
    ctx = X448PrivateKey.from_private_bytes(esk).public_key().public_bytes_raw()
    ssx = _openssl(esk, pkx)
    ctm, ssm = oracle.kyber_kem_encaps(k, ek, ee[56:])
    return pk, sk, ctx + ctm, ssx + ssm


@pytest.mark.parametrize("name,k", [("Kyber768-X448", 3), ("Kyber1024-X448", 4)])
def test_hybrid_x448_from_parts(name, k):
    assert ox.hybrid_seed_sizes(name) == (88, 56)
    pksz, sksz, ctsz = ox.hybrid_sizes(name)
    assert (pksz, sksz, ctsz) == {3: (1240, 2456, 1144), 4: (1624, 3224, 1624)}[k]
    for i in range(4):
        seed = hashlib.shake_256(b"s%d" % i + name.encode()).digest(64)
        eseed = hashlib.shake_256(b"e%d" % i + name.encode()).digest(56)
        pk, sk, ct, ss = _hybrid_from_parts(name, k, seed, eseed)
        assert ox.hybrid_keygen(name, seed) == (pk, sk)
        assert ox.hybrid_encaps(name, pk, eseed) == (ct, ss, 0)
        assert ox.hybrid_decaps(name, sk, ct) == (ss, 0)
    # a low-order X448 share is kem.ErrPubKey on both sides (xkem.go:150-156)
    low = _le(1)
    assert ox.hybrid_encaps(name, low + pk[56:], eseed)[2] == 1
    assert ox.hybrid_decaps(name, sk, low + ct[56:])[1] == 1


def test_device_x448_limb_arithmetic_on_host(tmp_path):
    """csrc/x448.cuh compiled as plain C++ (CUDA qualifiers defined away): field operations on edge values and at the
    accumulator bound, the fold, and the ladder and low-order test against the oracle."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    ox.build()
    exe = str(tmp_path / "x448_limbs")
    r = subprocess.run(["g++", "-O2", "-std=c++17", os.path.join(root, "tests", "cpp", "test_x448_limbs.cpp"), "-o", exe,
                        os.path.join(root, "oracle", "liboracle_x448.so"), os.path.join(root, "oracle", "liboracle.so"),
                        "-Wl,-rpath," + os.path.join(root, "oracle")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "bad=0" in r.stdout, r.stdout
