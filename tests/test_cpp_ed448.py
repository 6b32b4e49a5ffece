"""The Ed448 and Ed448-Dilithium3 entries of the C++ sign::Scheme (include/circl_b200.hpp), through
tests/cpp/test_sign_ed448.cpp: their registry and sizes on the CPU, transcripts against OpenSSL and the oracle on the
GPU."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build(tmp_path):
    from circl_b200 import _ffi
    _ffi.lib()
    exe = str(tmp_path / "test_sign_ed448")
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "cpp", "test_sign_ed448.cpp"), "-o", exe,
           "-L", os.path.join(ROOT, "circl_b200"), "-lcirclb200", "-Wl,-rpath," + os.path.join(ROOT, "circl_b200")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_registry_and_sizes(tmp_path):
    exe = _build(tmp_path)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120, env=dict(os.environ, CB200_SIZES_ONLY="1"))
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_transcripts_match_openssl_and_oracle(tmp_path):
    from cryptography.hazmat.primitives.asymmetric.ed448 import Ed448PrivateKey
    from oracle import ed448 as oe
    exe = _build(tmp_path)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout + r.stderr
    blocks, cur, pending = {}, None, {}
    for line in r.stdout.splitlines():
        if line.startswith("scheme="):
            cur = line.split("=", 1)[1]
            blocks[cur] = dict(pending)
            pending = {}
        elif "=" in line:
            k, v = line.split("=", 1)
            (pending if k == "ctxsig" else blocks[cur])[k] = bytes.fromhex(v)
    seed = bytes((5 * i + 2) & 0xFF for i in range(57))
    b = blocks["Ed448"]
    k = Ed448PrivateKey.from_private_bytes(seed)
    assert b["pk"] == k.public_key().public_bytes_raw() and b["sk"] == seed + b["pk"]
    assert b["sig"] == k.sign(b"hello")
    assert b["ctxsig"] == oe.ed448_sign(b["sk"], b"hello", b"ctx")
    b = blocks["Ed448-Dilithium3"]
    pk, sk = oe.eddilithium3_keygen(seed)
    assert (b["pk"], b["sk"]) == (pk, sk)
    assert b["sig"] == oe.eddilithium3_sign(sk, b"hello")
