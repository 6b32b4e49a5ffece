"""The lane mapping of the noise that the K-PKE kernels sample themselves (csrc/kyber.cuh noise_select / noise_cbd),
compiled as host code (nvcc, no GPU): for random SHAKE256 outputs, lane v's coefficients equal the oracle's CBD2 and
CBD3 polynomials at indices 16 s + 2 v + b (tests/cpp/test_noise_octet.cu)."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_noise_octet_mapping_on_host(tmp_path):
    import oracle
    oracle.build()
    exe = str(tmp_path / "noise_octet")
    odir = os.path.join(ROOT, "oracle")
    r = subprocess.run([os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc"), "-O2", "-std=c++17", "--expt-relaxed-constexpr",
                        "-Wno-deprecated-gpu-targets", os.path.join(ROOT, "tests", "cpp", "test_noise_octet.cu"), "-o", exe,
                        "-L", odir, "-loracle", "-Xlinker", "-rpath=" + odir], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "bad=0" in r.stdout, r.stdout[-2000:]
