"""DHKEM(P-384, HKDF-SHA384) and DHKEM(P-521, HKDF-SHA512) of the C++ kem::Scheme (include/circl_b200.hpp) through
tests/cpp/test_kem_nistp.cpp: the kem::p384 / kem::p521 registries, sizes, key checks and argument errors, with
kem::All(), kem::hpke::All() and kem::p256::All() unchanged, on the CPU; round trips and invalid keys on the GPU, with
the RFC 9180 vectors of both mode families for P-521 and the hashlib / OpenSSL model for P-384."""
import os
import random
import subprocess

import pytest

from conftest import load_golden
from nistp_model import CURVES
import nistp_model as model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    from circl_b200 import _ffi
    _ffi.lib()
    path = str(tmp_path_factory.mktemp("kem_nistp") / "test_kem_nistp")
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "cpp", "test_kem_nistp.cpp"), "-o", path,
           "-L", os.path.join(ROOT, "circl_b200"), "-lcirclb200", "-Wl,-rpath," + os.path.join(ROOT, "circl_b200")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return path


@pytest.mark.parametrize("bits", [384, 521])
def test_registry_and_sizes(exe, bits):
    r = subprocess.run([exe, str(bits)], capture_output=True, text=True, timeout=120,
                       env=dict(os.environ, CB200_SIZES_ONLY="1"))
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout + r.stderr


def _run(exe, bits, lines):
    r = subprocess.run([exe, str(bits)], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout + r.stderr
    out = [ln for ln in r.stdout.splitlines() if ln.startswith("pk=")]
    assert len(out) == len(lines)
    return [dict(kv.split("=") for kv in ln.split()) for ln in out]


@pytest.mark.gpu
def test_p521_rfc_vectors(exe):
    vs = load_golden("hpke_p521_vectors.json.gz")["vectors"]
    picks = [v for v in vs if v["mode"] in (0, 2)]
    lines = [f"base {v['ikmR']} {v['ikmE']}" if v["mode"] == 0 else f"auth {v['ikmR']} {v['ikmS']} {v['ikmE']}"
             for v in picks]
    for v, got in zip(picks, _run(exe, 521, lines)):
        assert got == {"pk": v["pkRm"], "enc": v["enc"], "ss": v["shared_secret"], "dec": v["shared_secret"]}


@pytest.mark.gpu
def test_p384_against_the_model(exe):
    c = CURVES[384]
    rng = random.Random(384)
    ikm = [bytes(rng.randrange(256) for _ in range(c.nbytes)) for _ in range(12)]
    lines = [f"base {ikm[i].hex()} {ikm[i + 1].hex()}" if i % 6 == 0 else
             f"auth {ikm[i].hex()} {ikm[i + 1].hex()} {ikm[i + 2].hex()}" for i in (0, 3, 6, 9)]
    for ln, got in zip(lines, _run(exe, 384, lines)):
        parts = [bytes.fromhex(h) for h in ln.split()[1:]]
        pkR, _ = model.derive_key_pair(c, parts[0])
        skS = model.derive_key_pair(c, parts[1])[1] if len(parts) == 3 else None
        enc, ss = model.encaps(c, pkR, parts[-1], skS)
        assert got == {"pk": pkR.hex(), "enc": enc.hex(), "ss": ss.hex(), "dec": ss.hex()}
