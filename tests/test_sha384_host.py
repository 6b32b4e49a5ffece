"""circl_b200/csrc/sha2.cuh's SHA-384 and two-block labeled HKDF-Expand compiled for the host (g++, no GPU) through
tests/cpp/test_sha384_host.cpp, against hashlib / hmac: SHA-384 and HMAC-SHA384 (with a one-digest key and with the
constant pads of the all-zero salt) over every message length 0..300, LabeledExtract for kem_id 0x11 (SHA-384) and 0x12
(SHA-512), and LabeledExpand's first two blocks T(1) || T(2) as P-521's 66-byte DeriveKeyPair candidate needs them."""
import hashlib
import hmac
import os
import random
import subprocess

import pytest

from nistp_model import CURVES, labeled_expand, labeled_extract

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def run(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("sha384") / "sha384_host")
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", os.path.join(ROOT, "tests", "cpp", "test_sha384_host.cpp"),
                        "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]

    def go(lines):
        out = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stderr
        res = out.stdout.splitlines()
        assert len(res) == len(lines)
        return res
    return go


def _h(b):
    return b.hex() if b else "-"


def test_sha384_and_hmac(run):
    rng = random.Random(384)
    msgs = [bytes(rng.randrange(256) for _ in range(n)) for n in range(301)]
    key = bytes(rng.randrange(256) for _ in range(48))
    lines = [f"sha384 {_h(m)}" for m in msgs] + [f"hmac384 {key.hex()} {_h(m)}" for m in msgs]
    lines += [f"hmac384 - {_h(m)}" for m in msgs[::7]]
    want = [hashlib.sha384(m).hexdigest() for m in msgs] + [hmac.new(key, m, hashlib.sha384).hexdigest() for m in msgs]
    want += [hmac.new(bytes(48), m, hashlib.sha384).hexdigest() for m in msgs[::7]]
    assert run(lines) == want


@pytest.mark.parametrize("bits", [384, 521])
def test_labeled_extract_and_two_block_expand(run, bits):
    c = CURVES[bits]
    rng = random.Random(bits)
    lines, want = [], []
    for n in (0, 1, c.nbytes, 2 * c.nbytes, 3 * c.npk):
        ikm = bytes(rng.randrange(256) for _ in range(n))
        lines.append(f"extract {c.kem_id:x} dkp_prk {_h(ikm)}")
        want.append(labeled_extract(c, b"", b"dkp_prk", ikm).hex())
    for info, L in ((b"\x00", c.nbytes), (b"\x07", 66), (b"\xff", 2 * c.nss), (bytes(range(40)), 2 * c.nss - 1)):
        prk = bytes(rng.randrange(256) for _ in range(c.nss))
        lines.append(f"expand2 {c.kem_id:x} {prk.hex()} candidate {info.hex()} {L}")
        t = labeled_expand(c, prk, b"candidate", info, L)
        # the driver prints the whole of T(1) || T(2); the first L bytes are LabeledExpand's output
        full = labeled_expand(c, prk, b"candidate", info, 2 * c.nss) if L == 2 * c.nss else None
        want.append((full or t).hex())
    res = run(lines)
    assert res[:5] == want[:5]
    for r, w in zip(res[5:], want[5:]):
        assert r[:len(w)] == w
