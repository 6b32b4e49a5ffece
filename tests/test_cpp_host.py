"""The compiled host-side mirror (include/circl_b200.hpp): it must compile against the header (CPU),
and on the GPU its transcripts must equal the oracle's for the same seeds."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_exe(out_dir):
    """Link tests/cpp/test_scheme.cpp against the library into out_dir: the source tree may be read-only."""
    from circl_b200 import _ffi
    assert os.path.exists(_ffi.LIB_PATH)
    exe = os.path.join(str(out_dir), "test_scheme")
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "cpp", "test_scheme.cpp"), "-o", exe,
           "-L", os.path.join(ROOT, "circl_b200"), "-lcirclb200", "-Wl,-rpath," + os.path.join(ROOT, "circl_b200")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_cpp_host_layer_compiles_and_links(tmp_path):
    build_exe(tmp_path)


@pytest.mark.gpu
def test_cpp_host_layer_matches_oracle(tmp_path):
    import oracle
    exe = build_exe(tmp_path)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "ALL OK" in r.stdout
    blocks, cur = {}, None
    for line in r.stdout.splitlines():
        if line.startswith("scheme="):
            cur = line.split("=", 1)[1]
            blocks[cur] = {}
        elif "=" in line and cur:
            k, v = line.split("=", 1)
            blocks[cur][k] = bytes.fromhex(v)
    for name, k in (("ML-KEM-512", 2), ("ML-KEM-768", 3), ("ML-KEM-1024", 4)):
        seed = bytes((i * 7 + k) & 0xFF for i in range(64))
        eseed = bytes(255 - i for i in range(32))
        ek, dk = oracle.mlkem_keygen(k, seed)
        ct, ss = oracle.mlkem_encaps(k, ek, eseed)
        b = blocks[name]
        assert (b["ek"], b["dk"], b["ct"], b["ss"]) == (ek, dk, ct, ss)
        bad = bytearray(ct)
        bad[3] ^= 1
        assert b["ss_rejected"] == oracle.mlkem_decaps(k, dk, bytes(bad))
    dseed = bytes((3 * i + 1) & 0xFF for i in range(32))
    pk, sk = oracle.mldsa65_keygen(dseed)
    b = blocks["ML-DSA-65"]
    assert (b["pk"], b["sk"]) == (pk, sk)
    assert b["sig"] == oracle.mldsa65_sign(sk, b"hello", ctx=b"ctx")[0]
    for name, k in (("Kyber512", 2), ("Kyber768", 3), ("Kyber1024", 4)):
        seed = bytes((i * 11 + k) & 0xFF for i in range(64))
        eseed = bytes(i ^ 0x5A for i in range(32))
        ek, dk = oracle.kyber_kem_keygen(k, seed)
        b = blocks[name]
        assert (b["ek"], b["dk"]) == (ek, dk)
        assert (b["ct"], b["ss"]) == oracle.kyber_kem_encaps(k, ek, eseed)
    pk, sk = oracle.mldsa_keygen(3, dseed)
    b = blocks["Dilithium3"]
    assert (b["pk"], b["sk"]) == (pk, sk)
    assert b["sig"] == oracle.mldsa_sign(3, sk, b"hello")[0]
    hseed64, hseed32 = bytes((i * 5 + 3) & 0xFF for i in range(64)), bytes((i * 5 + 3) & 0xFF for i in range(32))
    e32, e64 = bytes((i * 9 + 1) & 0xFF for i in range(32)), bytes((i * 9 + 1) & 0xFF for i in range(64))
    b = blocks["X-Wing"]
    assert (b["pk"], b["sk"]) == (oracle.xwing_keygen(hseed32), hseed32)
    assert (b["ct"], b["ss"]) == oracle.xwing_encaps(b["pk"], e64)
    for name in ("X25519MLKEM768", "Kyber768-X25519", "Kyber512-X25519"):
        b = blocks[name]
        assert (b["pk"], b["sk"]) == oracle.hybrid_keygen(name, hseed64)
        assert (b["ct"], b["ss"], 0) == oracle.hybrid_encaps(name, b["pk"], e32)


def test_kyber_low_format_fast_path_on_host(tmp_path):
    """csrc/kyber.cuh's low-format fast path compiled as host code (nvcc, no GPU): the Shoup-form Montgomery product
    against montReduce for every twiddle and every int16, barrett_lo on every int16, and an emulated octet (the
    kernels' own pass and transposition functions, lane after lane) against nttGeneric / invNTTGeneric on inputs up
    to the bounds of the fast range, plus the range predicate (tests/cpp/test_kyber_low.cu)."""
    import oracle
    oracle.build()
    exe = str(tmp_path / "kyber_low")
    odir = os.path.join(ROOT, "oracle")
    r = subprocess.run([os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc"), "-O2", "-std=c++17", "--expt-relaxed-constexpr", "-Wno-deprecated-gpu-targets",
                        os.path.join(ROOT, "tests", "cpp", "test_kyber_low.cu"), "-o", exe, "-L", odir, "-loracle",
                        "-Xlinker", "-rpath=" + odir], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "bad=0" in r.stdout, r.stdout[-2000:]


def test_dilithium_shoup_constants_on_host(tmp_path):
    """csrc/dilithium.cuh's Shoup-form multiplication by a constant (every forward / inverse twiddle and ROver256)
    against the oracle's montReduceLe2Q, compiled as host code (tests/cpp/test_dil_shoup.cu)."""
    import oracle
    oracle.build()
    exe = str(tmp_path / "dil_shoup")
    odir = os.path.join(ROOT, "oracle")
    r = subprocess.run([os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc"), "-O2", "-std=c++17", "--expt-relaxed-constexpr",
                        "-Wno-deprecated-gpu-targets", os.path.join(ROOT, "tests", "cpp", "test_dil_shoup.cu"), "-o", exe,
                        "-L", odir, "-loracle", "-Xlinker", "-rpath=" + odir], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "bad=0" in r.stdout, r.stdout[-2000:]


def test_dilithium_transform_passes_on_host(tmp_path):
    """csrc/dilithium.cuh's transform passes compiled as host code: an emulated octet (S-layout pass with immediate
    Shoup pairs, padded-tile transposition, C-layout pass reading the lane-transposed staged pairs) against the
    oracle's NTT / InvNTT, unnormalised, on arbitrary uint32 inputs (tests/cpp/test_dil_passes.cu)."""
    import oracle
    oracle.build()
    exe = str(tmp_path / "dil_passes")
    odir = os.path.join(ROOT, "oracle")
    r = subprocess.run([os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc"), "-O2", "-std=c++17", "--expt-relaxed-constexpr",
                        "-Wno-deprecated-gpu-targets", os.path.join(ROOT, "tests", "cpp", "test_dil_passes.cu"), "-o", exe,
                        "-L", odir, "-loracle", "-Xlinker", "-rpath=" + odir], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "bad=0" in r.stdout, r.stdout[-2000:]
