"""circl_b200/csrc/frodo.cuh compiled for the host (g++, no GPU) through tests/cpp/test_frodo_host.cpp: the sampler on
all 65536 inputs, 15-bit pack / unpack and message encode / decode against the oracle (oracle/frodo.c), and the masks of
the constant-time compare."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def run(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("frodo") / "frodo_host")
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", os.path.join(ROOT, "tests", "cpp", "test_frodo_host.cpp"),
                        "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]

    def go(lines):
        out = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stderr
        res = out.stdout.splitlines()
        assert len(res) == len(lines)
        return res
    return go


@pytest.fixture(scope="module")
def O():
    from oracle import frodo as oracle_frodo
    return oracle_frodo


def test_sampler_every_input(run, O):
    got = np.frombuffer(bytes.fromhex(run(["sample -"])[0]), dtype=">u2")
    want = np.array([O.sample(r) for r in range(65536)], dtype=np.uint16)
    assert np.array_equal(got, want)
    assert set(np.where(want < 0x8000, want, want.astype(np.int64) - 0x10000).tolist()) <= set(range(-12, 13))


def test_pack_unpack(run, O):
    rng = np.random.default_rng(1)
    vals = np.concatenate([rng.integers(0, 65536, size=(300, 8)), np.full((1, 8), 0xFFFF), np.zeros((1, 8), int),
                           np.full((1, 8), 0x7FFF)]).astype(np.uint16)
    got = run([f"pack {v.astype('<u2').tobytes().hex()}" for v in vals])
    assert got == [O.pack(v).hex() for v in vals]
    back = run([f"unpack {g}" for g in got])
    assert [np.frombuffer(bytes.fromhex(b), "<u2").tolist() for b in back] == [(v & 0x7FFF).tolist() for v in vals]
    raw = [rng.bytes(15) for _ in range(200)]
    got = run([f"unpack {r.hex()}" for r in raw])
    assert [np.frombuffer(bytes.fromhex(g), "<u2").tolist() for g in got] == [O.unpack(r).tolist() for r in raw]


def test_encode_decode(run):
    import frodo_model as M
    rng = np.random.default_rng(2)
    msgs = [rng.bytes(16) for _ in range(100)] + [bytes(16), b"\xff" * 16]
    got = run([f"encode {m.hex()}" for m in msgs])
    assert [np.frombuffer(bytes.fromhex(g), "<u2").tolist() for g in got] == [M.encode(m).tolist() for m in msgs]
    # decode of noisy encodings, including every residue near the rounding boundaries
    ws = [(M.encode(m) + rng.integers(-4095, 4096, size=64)) & 0xFFFF for m in msgs]
    ws.append(np.arange(64, dtype=np.int64) * 1024 + 4095)
    got = run([f"decode {w.astype('<u2').tobytes().hex()}" for w in ws])
    assert got == [M.decode(w).hex() for w in ws]
    assert got[:len(msgs)] == [m.hex() for m in msgs]


def test_compare_masks(run):
    vals = [0, 1, 2, 0x7FFF, 0x8000, 0xFFFF, 0x10000, 0xFFFFFFFF]
    got = run([f"mask {v}" for v in vals])
    assert got == [("0 0" if v == 0 else "1 255") for v in vals]
