"""The C++ blindrsa mirror (include/circl_b200.hpp) through tests/cpp/test_brsa.cpp: key, variant and size errors on
the CPU; on the GPU, the four RFC 9474 vectors (blind_sig from blinded_msg, sig verifying), a batch under every fixture
key against tests/brsa_model.py with an edge row failing only its own op, and a tampered signature."""
import os
import random
import subprocess

import pytest

import brsa_model as bm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    from circl_b200 import _ffi
    _ffi.lib()
    path = str(tmp_path_factory.mktemp("brsa_cpp") / "test_brsa")
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "cpp", "test_brsa.cpp"), "-o", path,
           "-L", os.path.join(ROOT, "circl_b200"), "-lcirclb200", "-Wl,-rpath," + os.path.join(ROOT, "circl_b200")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return path


def _hx(x):
    return x.to_bytes((x.bit_length() + 7) // 8 or 1, "big").hex()


def _fields(k):
    return [_hx(v) for v in (k.n, k.e, k.p, k.q, *k.crt())]


def test_key_variant_and_size_errors(exe):
    r = subprocess.run([exe, *_fields(bm.pem_key())], capture_output=True, text=True, timeout=120,
                       env=dict(os.environ, CB200_SIZES_ONLY="1"))
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_vectors_and_model_parity(exe):
    lines, want = [], []
    k = bm.rfc_key()
    for variant, v in enumerate(bm.rfc_vectors()):
        lines.append("sign " + " ".join(_fields(k)) + " " + v["blinded_msg"])
        want.append("sig=" + v["blind_sig"])
        lines.append(f"verify {variant} {_hx(k.n)} {_hx(k.e)} {v['sig']} {v['input_msg']}")
        want.append("ok")
    for name, k in bm.all_keys().items():
        rng = random.Random(name)
        cs = [rng.randrange(k.n) for _ in range(5)] + [k.n]
        rows = b"".join(bm.i2osp(c, k.klen) for c in cs)
        lines.append("sign " + " ".join(_fields(k)) + " " + rows.hex())
        res = [bm.blind_sign(k, bm.i2osp(c, k.klen)) for c in cs]
        want.append("err=internal st=" + bytes(r[0] for r in res).hex())
        lines.append("sign " + " ".join(_fields(k)) + " " + rows[:-k.klen].hex())
        want.append("sig=" + b"".join(r[1] for r in res[:-1]).hex())
        msgs = [rng.randbytes(rng.randrange(200)) or b"x" for _ in range(3)]
        sigs = [bm.tampered(k, 0, m, rng)[0][1] for m in msgs]
        lines.append(f"verify 3 {_hx(k.n)} {_hx(k.e)} {b''.join(sigs).hex()} " + " ".join(m.hex() for m in msgs))
        want.append("ok")
        sigs[1] = bm.tampered(k, 0, msgs[1], rng)[1][1]  # trailer
        lines.append(f"verify 1 {_hx(k.n)} {_hx(k.e)} {b''.join(sigs).hex()} " + " ".join(m.hex() for m in msgs))
        want.append("err=verification st=000200")
    r = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout + r.stderr
    assert r.stdout.splitlines()[:-1] == want
