"""DHKEM(P-256, HKDF-SHA256) of the C++ kem::Scheme (include/circl_b200.hpp) through tests/cpp/test_kem_p256.cpp: the
kem::p256 registry, sizes, key checks and argument errors, with kem::All() and kem::hpke::All() unchanged, on the CPU;
round trips, invalid keys and the RFC 9180 vectors of both mode families (Encap / AuthEncap) on the GPU."""
import os
import subprocess

import pytest

from conftest import load_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build(tmp_path):
    from circl_b200 import _ffi
    _ffi.lib()
    exe = str(tmp_path / "test_kem_p256")
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "cpp", "test_kem_p256.cpp"), "-o", exe,
           "-L", os.path.join(ROOT, "circl_b200"), "-lcirclb200", "-Wl,-rpath," + os.path.join(ROOT, "circl_b200")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_registry_and_sizes(tmp_path):
    exe = _build(tmp_path)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120, env=dict(os.environ, CB200_SIZES_ONLY="1"))
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_round_trips_and_rfc_vectors(tmp_path):
    exe = _build(tmp_path)
    vs = load_golden("hpke_p256_vectors.json.gz")["vectors"]
    picks = [v for v in vs if v["mode"] in (0, 2)]
    lines = [f"base {v['ikmR']} {v['ikmE']}" if v["mode"] == 0 else f"auth {v['ikmR']} {v['ikmS']} {v['ikmE']}"
             for v in picks]
    r = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout + r.stderr
    out = [ln for ln in r.stdout.splitlines() if ln.startswith("pk=")]
    assert len(out) == len(picks)
    for v, ln in zip(picks, out):
        got = dict(kv.split("=") for kv in ln.split())
        assert got == {"pk": v["pkRm"], "enc": v["enc"], "ss": v["shared_secret"], "dec": v["shared_secret"]}
