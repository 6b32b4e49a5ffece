"""Builds circl_b200/libcirclb200.so in-tree with nvcc for sm_90a (no JIT, no torch)."""
from __future__ import annotations

import concurrent.futures as cf
import glob
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libcirclb200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v",
]


def _deps_digest() -> str:
    h = hashlib.sha256()
    for f in sorted(glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(CSRC, "*.h"))
                    + glob.glob(os.path.join(HERE, "..", "include", "*.h"))):
        h.update(open(f, "rb").read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def _compile(src: str, digest: str, verbose: bool) -> str:
    name = os.path.splitext(os.path.basename(src))[0]
    obj = os.path.join(OBJ, name + ".o")
    stamp = obj + ".stamp"
    want = hashlib.sha256(open(src, "rb").read() + digest.encode()).hexdigest()
    if os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == want:
        return obj
    r = subprocess.run([NVCC, *FLAGS, "-c", src, "-o", obj], capture_output=True, text=True)
    log = os.path.join(OBJ, name + ".ptxas.log")
    open(log, "w").write(r.stdout + r.stderr)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    if verbose:
        sys.stderr.write(f"[build] {name}.cu ok\n")
    open(stamp, "w").write(want)
    return obj


def build_library(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    srcs = sorted(glob.glob(os.path.join(CSRC, "*.cu")))
    digest = _deps_digest() + ("force" + os.urandom(4).hex() if force else "")
    with cf.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(lambda s: _compile(s, digest, verbose), srcs))
    newest = max(os.path.getmtime(o) for o in objs)
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < newest:
        r = subprocess.run([NVCC, "-shared", "-o", LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a",
                            "-cudart", "static"], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    print(build_library(force="--force" in sys.argv, verbose=True))
