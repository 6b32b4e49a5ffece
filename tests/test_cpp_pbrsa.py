"""The C++ partiallyblindrsa mirror (include/circl_b200.hpp) through tests/cpp/test_pbrsa.cpp: key and size errors on
the CPU (a key whose primes are not safe among them); on the GPU, a batch under every fixture key against
tests/pbrsa_model.py with per-op metadata and an edge row failing only its own op, and Verify with a swapped
metadata string."""
import os
import random
import subprocess

import pytest

import brsa_model as bm
import pbrsa_model as pm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    from circl_b200 import _ffi
    _ffi.lib()
    path = str(tmp_path_factory.mktemp("pbrsa_cpp") / "test_pbrsa")
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "cpp", "test_pbrsa.cpp"), "-o", path,
           "-L", os.path.join(ROOT, "circl_b200"), "-lcirclb200", "-Wl,-rpath," + os.path.join(ROOT, "circl_b200")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return path


def _hx(x):
    return x.to_bytes((x.bit_length() + 7) // 8 or 1, "big").hex()


def _fields(k):
    return [_hx(v) for v in (k.n, k.p, k.q, pow(k.q, -1, k.p))]


def test_key_and_size_errors(exe):
    weak = bm.all_keys()["rsa2048u"]  # primes = 3 mod 4, not safe
    assert weak.p % 4 == 3 and weak.q % 4 == 3
    r = subprocess.run([exe, *_fields(pm.keys()["strong2048"]), *_fields(weak)], capture_output=True, text=True,
                       timeout=120, env=dict(os.environ, CB200_SIZES_ONLY="1"))
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_model_parity(exe):
    lines, want = [], []
    for name, k in pm.keys().items():
        rng = random.Random(name)
        metas = [b"", b"a", rng.randbytes(130), rng.randbytes(7), rng.randbytes(40)]
        cs = [rng.randrange(k.n) for _ in range(4)] + [k.n]
        rows = b"".join(bm.i2osp(c, k.klen) for c in cs)
        res = [pm.blind_sign(k, bm.i2osp(c, k.klen), m) for c, m in zip(cs, metas)]
        lines.append("sign " + " ".join(_fields(k)) + " " + rows.hex() + " " + " ".join(m.hex() or "-" for m in metas))
        want.append("err=internal st=" + bytes(r[0] for r in res).hex())
        lines.append("sign " + " ".join(_fields(k)) + " " + rows[:-k.klen].hex() + " " +
                     " ".join(m.hex() or "-" for m in metas[:-1]))
        want.append("sig=" + b"".join(r[1] for r in res[:-1]).hex())
        msgs = [rng.randbytes(rng.randrange(200)) for _ in range(3)]
        sigs = [pm.sign(k, m, md, rng) for m, md in zip(msgs, metas)]
        pairs = " ".join(f"{m.hex() or '-'} {md.hex() or '-'}" for m, md in zip(msgs, metas))
        lines.append(f"verify {_hx(k.n)} {b''.join(sigs).hex()} {pairs}")
        want.append("ok")
        swapped = [metas[0], metas[2], metas[1]]
        pairs = " ".join(f"{m.hex() or '-'} {md.hex() or '-'}" for m, md in zip(msgs, swapped))
        lines.append(f"verify {_hx(k.n)} {b''.join(sigs).hex()} {pairs}")
        want.append("err=verification st=000202")
    r = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout + r.stderr
    assert r.stdout.splitlines()[:-1] == want
