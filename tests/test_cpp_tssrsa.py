"""The C++ tssrsa mirror (include/circl_b200.hpp) through tests/cpp/test_tssrsa.cpp: size and argument errors on the
CPU; on the GPU, signature shares under two fixture keys and a Combine batch with an honest, a corrupted and an
index-0 op, each against tests/tssrsa_model.py."""
import os
import random
import subprocess

import pytest

import brsa_model as bm
import tssrsa_model as tm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    from circl_b200 import _ffi
    _ffi.lib()
    path = str(tmp_path_factory.mktemp("tssrsa_cpp") / "test_tssrsa")
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "cpp", "test_tssrsa.cpp"), "-o", path,
           "-L", os.path.join(ROOT, "circl_b200"), "-lcirclb200", "-Wl,-rpath," + os.path.join(ROOT, "circl_b200")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return path


def _hx(x, n=None):
    return x.to_bytes(n or (x.bit_length() + 7) // 8 or 1, "big").hex()


def test_size_and_argument_errors(exe):
    k = bm.all_keys()["rsa2048"]
    r = subprocess.run([exe, _hx(k.n), _hx(k.e)], capture_output=True, text=True, timeout=120,
                       env=dict(os.environ, CB200_SIZES_ONLY="1"))
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout + r.stderr


class _Stream:
    def __init__(self, rng):
        self.rng = rng

    def read(self, n):
        return self.rng.randbytes(n)


@pytest.mark.gpu
def test_model_parity(exe):
    lines, want = [], []
    for name in ("rsa2048", "rsa3073"):
        k = bm.all_keys()[name]
        kl, players, threshold = k.klen, 5, 3
        rng = random.Random(name)
        s = tm.deal(_Stream(rng), players, threshold, k.p, k.q, k.e)
        E = [2 * tm.delta(players) * v for v in s]
        xs = [rng.randrange(k.n) for _ in range(4)] + [0, k.n]
        rows = b"".join(x.to_bytes(kl, "big") for x in xs)
        lines.append(f"sign {_hx(k.n)} {players} {_hx(E[1])} {rows.hex()}")
        want.append("xi=" + b"".join(pow(x, E[1], k.n).to_bytes(kl, "big") for x in xs).hex())
        S = [1, 3, 4]
        xi = [[pow(x, E[j - 1], k.n) for j in S] for x in xs[:3]]
        xi[1][2] ^= 1  # a corrupted share fails its own op only
        blob = b"".join(v.to_bytes(kl, "big") for op in xi for v in op)
        msgs = b"".join(x.to_bytes(kl, "big") for x in xs[:3])
        res = [tm.combine(k.n, k.e, players, S, xi[i], xs[i]) for i in range(3)]
        lines.append(f"combine {_hx(k.n)} {_hx(k.e)} {players} {threshold} 3 {','.join(map(str, S))} {blob.hex()} "
                     f"{msgs.hex()}")
        want.append("err=internal st=" + bytes(r[0] for r in res).hex())
        lines.append(f"combine {_hx(k.n)} {_hx(k.e)} {players} {threshold} 3 {','.join(map(str, S))} "
                     f"{blob[:3 * kl].hex()} {msgs[:kl].hex()}")
        want.append("sig=" + _hx(res[0][1], kl))
        lines.append(f"combine {_hx(k.n)} {_hx(k.e)} {players} {threshold} 3 0,3,4 {blob[:3 * kl].hex()} "
                     f"{msgs[:kl].hex()}")
        want.append("err=calc st=01")
    r = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout + r.stderr
    assert r.stdout.splitlines()[:-1] == want
