"""circl_b200/csrc/sha2.cuh compiled for the host (g++, no GPU) through tests/cpp/test_sha2_host.cpp: SHA-256,
HMAC-SHA256 / HMAC-SHA512 (with a one-digest key and with the constant pads of the all-zero salt) and HPKE's labeled
Extract / Expand against hashlib / hmac, over every message length 0..300 and at the sizes the HPKE kernels use."""
import hashlib
import hmac
import os
import random
import subprocess

import pytest

import hpke_model as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def run(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("sha2") / "sha2_host")
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", os.path.join(ROOT, "tests", "cpp", "test_sha2_host.cpp"),
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


def _msgs(seed):
    rng = random.Random(seed)
    return [bytes(rng.randrange(256) for _ in range(n)) for n in range(301)]


def test_sha256_every_length(run):
    ms = _msgs(1)
    assert run([f"sha256 {_h(m)}" for m in ms]) == [hashlib.sha256(m).hexdigest() for m in ms]


@pytest.mark.parametrize("op,h,klen", [("hmac256", hashlib.sha256, 32), ("hmac512", hashlib.sha512, 64)])
def test_hmac_every_length(run, op, h, klen):
    ms = _msgs(klen)
    rng = random.Random(op)
    keys = [bytes(rng.randrange(256) for _ in range(klen)) for _ in ms]
    got = run([f"{op} {k.hex()} {_h(m)}" for k, m in zip(keys, ms)])
    assert got == [hmac.new(k, m, h).hexdigest() for k, m in zip(keys, ms)]
    # the all-zero salt of LabeledExtract, through the precomputed pad states
    got = run([f"{op} - {_h(m)}" for m in ms])
    assert got == [hmac.new(bytes(klen), m, h).hexdigest() for m in ms]


@pytest.mark.parametrize("kid", [M.X25519_ID, M.X448_ID])
def test_labeled_functions_at_kernel_sizes(run, kid):
    m = M.KEMS[kid]
    n, nh = m.n, m.nh
    rng = random.Random(kid)
    rb = lambda k: bytes(rng.randrange(256) for _ in range(k))  # noqa: E731
    lines, want = [], []
    for _ in range(20):
        # DeriveKeyPair: Extract(dkp_prk, seed), Expand(sk, "", Nsk)
        seed, prk = rb(n), rb(nh)
        lines.append(f"extract {kid:x} {b'dkp_prk'.hex()} {seed.hex()}")
        want.append(m.extract(b"", b"dkp_prk", seed).hex())
        lines.append(f"expand {kid:x} {prk.hex()} {b'sk'.hex()} - - - {n}")
        want.append(m.expand(prk, b"sk", b"", n).hex())
        # ExtractAndExpand: dh of 1 or 2 keys, kem_context of 2 or 3 rows
        for nd, nc in ((1, 2), (2, 3)):
            dh, rows = rb(nd * n), [rb(n) for _ in range(nc)] + [b""] * (3 - nc)
            lines.append(f"extract {kid:x} {b'eae_prk'.hex()} {dh.hex()}")
            want.append(m.extract(b"", b"eae_prk", dh).hex())
            lines.append(f"expand {kid:x} {prk.hex()} {b'shared_secret'.hex()} {' '.join(_h(r) for r in rows)} {nh}")
            want.append(m.expand(prk, b"shared_secret", b"".join(rows), nh).hex())
    assert run(lines) == want


@pytest.mark.parametrize("kid", [M.X25519_ID, M.X448_ID])
def test_labeled_functions_every_length(run, kid):
    m = M.KEMS[kid]
    ms = _msgs(kid)
    prk = hashlib.sha512(b"prk").digest()[:m.nh]
    got = run([f"extract {kid:x} {b'lab'.hex()} {_h(x)}" for x in ms])
    assert got == [m.extract(b"", b"lab", x).hex() for x in ms]
    got = run([f"expand {kid:x} {prk.hex()} {b'info'.hex()} {_h(x[:len(x) // 3])} {_h(x[len(x) // 3:])} - {len(x) % m.nh + 1}"
               for x in ms[:280]])
    assert got == [m.expand(prk, b"info", x, len(x) % m.nh + 1).hex() for x in ms[:280]]
