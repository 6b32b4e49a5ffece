"""FrodoKEM-640-SHAKE through the C++ kem::Scheme (include/circl_b200.hpp) and tests/cpp/test_kem_frodo.cpp: the
kem::frodo registry, sizes and argument errors on the CPU (kem::All() keeps its twelve schemes); KeyGen, Encaps,
Decaps and a shared-key batch against the oracle on the GPU."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build(tmp_path):
    from circl_b200 import _ffi
    _ffi.lib()
    exe = str(tmp_path / "test_kem_frodo")
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "cpp", "test_kem_frodo.cpp"), "-o", exe,
           "-L", os.path.join(ROOT, "circl_b200"), "-lcirclb200", "-Wl,-rpath," + os.path.join(ROOT, "circl_b200")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_registry_and_sizes(tmp_path):
    exe = _build(tmp_path)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120, env=dict(os.environ, CB200_SIZES_ONLY="1"))
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_round_trips_against_oracle(tmp_path):
    from oracle import frodo as O
    exe = _build(tmp_path)
    rng = np.random.default_rng(21)
    cases = [(rng.bytes(48), rng.bytes(16)) for _ in range(3)]
    r = subprocess.run([exe], input="".join(f"{k.hex()} {e.hex()}\n" for k, e in cases), capture_output=True,
                       text=True, timeout=300)
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout + r.stderr
    out = [ln for ln in r.stdout.splitlines() if ln.startswith("pk=")]
    assert len(out) == len(cases)
    for (k, e), ln in zip(cases, out):
        pk, _ = O.keygen(k)
        _, ss = O.encaps(pk, e)
        assert dict(kv.split("=") for kv in ln.split()) == {"pk": pk[:32].hex(), "ss": ss.hex(), "dec": ss.hex()}
