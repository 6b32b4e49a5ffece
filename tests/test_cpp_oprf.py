"""The C++ oprf mirror (include/circl_b200.hpp) through tests/cpp/test_oprf.cpp: suites, sizes and argument errors on
the CPU; on the GPU, the three server types against the first RFC 9497 vector of every NIST suite and mode (DeriveKey,
Evaluate with the proof given r, FullEvaluate, VerifyFinalize), and Evaluate with the server's own randomness against
tests/oprf_model.py."""
import os
import subprocess

import pytest

import oprf_model as om
from conftest import load_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    from circl_b200 import _ffi
    _ffi.lib()
    path = str(tmp_path_factory.mktemp("oprf_cpp") / "test_oprf")
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "cpp", "test_oprf.cpp"), "-o", path,
           "-L", os.path.join(ROOT, "circl_b200"), "-lcirclb200", "-Wl,-rpath," + os.path.join(ROOT, "circl_b200")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return path


def test_suites_sizes_and_errors(exe):
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120, env=dict(os.environ, CB200_SIZES_ONLY="1"))
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_rfc9497_vectors_and_own_randomness(exe):
    lines, want = [], []
    for tv in load_golden("oprf_rfc9497.json.gz"):
        if tv["identifier"] not in om.SUITES:
            continue
        s, mode = om.SUITES[tv["identifier"]], tv["mode"]
        v = tv["vectors"][0]
        info = v.get("Info", "") or "-"
        r = v["Proof"]["r"] if "Proof" in v else "-"
        lines.append(f"vec {tv['identifier']} {mode} {tv['seed']} {tv['keyInfo']} {info} {r} {v['Input']} "
                     f"{v['BlindedElement']}")
        sk, pk = om.derive_key(s, mode, bytes.fromhex(tv["seed"]), bytes.fromhex(tv["keyInfo"]))
        want.append({"sk": tv["skSm"], "pk": pk.hex(), "ev": v["EvaluationElement"],
                     "proof": v["Proof"]["proof"] if "Proof" in v else "-", "out": v["Output"], "ok": "1"})
        if mode:
            lines.append(f"vec {tv['identifier']} {mode} {tv['seed']} {tv['keyInfo']} {info} - {v['Input']} "
                         f"{v['BlindedElement']}")
            want.append(dict(want[-1], proof="rand"))
    r = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout + r.stderr
    got = [dict(kv.split("=") for kv in ln.split()) for ln in r.stdout.splitlines() if ln.startswith("sk=")]
    assert got == want
