"""circl_b200/csrc/rsa.cuh compiled for the host (g++, no GPU) through tests/cpp/test_brsa_host.cpp, against Python
integers and tests/brsa_model.py: the Montgomery product and square at every word count with the operands 0, 1, m - 1
and the largest the reduction accepts (R - 1 times m - 1); exponentiation by random and all-ones exponents; BlindSign
(both CRT halves, Garner's recombination and the check) under every fixture key; and Verify on each EMSA-PSS failure
class."""
import os
import random
import subprocess

import pytest

import brsa_model as bm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORDS = [32, 48, 64, 96, 128]


@pytest.fixture(scope="module")
def run(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("brsa") / "brsa_host")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Wno-unknown-pragmas",
                        os.path.join(ROOT, "tests", "cpp", "test_brsa_host.cpp"), "-o", path],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]

    def go(lines):
        out = subprocess.run([path], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stderr
        res = out.stdout.splitlines()
        assert len(res) == len(lines)
        return res
    return go


def _h(x, w):
    return x.to_bytes(4 * w, "big").hex()


def _hx(x):
    """big-endian hex of x in whole bytes"""
    return x.to_bytes((x.bit_length() + 7) // 8 or 1, "big").hex()


def _modulus(w, rng, top):
    """an odd modulus of w words whose top word is `top` (small tops make R much larger than m)"""
    return (top << (32 * w - 32)) | rng.getrandbits(32 * w - 32) | 1


@pytest.mark.parametrize("w", WORDS)
def test_montgomery_product(run, w):
    rng = random.Random(w)
    R = 1 << (32 * w)
    lines, want = [], []
    for top in (0xffffffff, 0x80000000, 0x1234):
        m = _modulus(w, rng, top)
        ri = pow(R, -1, m)
        vals = [0, 1, m - 1, m - 2, rng.randrange(m), rng.randrange(m)]
        pairs = [(a, b) for a in vals for b in vals] + [(R - 1, m - 1), (m - 1, R - 1), (R - 1, 1)]
        for a, b in pairs:
            lines.append(f"mul {w} {_h(m, w)} {_h(a, w)} {_h(b, w)}")
            want.append(_h(a * b * ri % m, w))
    assert run(lines) == want


@pytest.mark.parametrize("w", WORDS)
def test_exponentiation(run, w):
    rng = random.Random(100 + w)
    lines, want = [], []
    for top in (0xffffffff, 0x80000000, 0x3):
        m = _modulus(w, rng, top)
        ones = (1 << m.bit_length()) - 1  # every window digit 15; exp_secret reads bitlen(m) bits
        for x in (0, 1, m - 1, rng.randrange(m)):
            for d in (0, 1, rng.randrange(m), ones >> 1, m - 1):
                lines.append(f"exps {w} {_h(m, w)} {_h(x, w)} {_h(d, w)}")
                want.append(_h(pow(x, d, m), w))
            for e in (3, 65537, 2**32 - 1, rng.randrange(3, 2**32) | 1):
                lines.append(f"expp {w} {_h(m, w)} {_h(x, w)} {e}")
                want.append(_h(pow(x, e, m), w))
        lines.append(f"exps {w} {_h(m, w)} {_h(7, w)} {_h(ones, w)}")  # d >= m still computes x^d (all windows 15)
        want.append(_h(pow(7, ones, m), w))
    assert run(lines) == want


def _classes(k):
    wp = next(w for w in (32, 48, 64) if max(k.p.bit_length(), k.q.bit_length()) <= 32 * w)
    wn = next(w for w in (64, 96, 128) if k.n.bit_length() <= 32 * w)
    return wp, wn


def _sign_line(k, c, crt=None):
    wp, wn = _classes(k)
    dp, dq, qinv = crt or k.crt()
    f = [k.n, k.e, k.p, k.q, dp, dq, qinv]
    return f"sign {wp} {wn} " + " ".join(map(_hx, f)) + " " + c.hex()


@pytest.mark.parametrize("name", ["rsa2048", "rsa3072", "rsa3073", "rsa2048e3", "rsa2048u", "rsa3000u", "rsa4096"])
def test_blind_sign(run, name):
    k = bm.all_keys()[name]
    rng = random.Random(name)
    cs = [0, 1, 2, k.n - 1, k.n, k.n + 1, (1 << (8 * k.klen)) - 1] + [rng.randrange(k.n) for _ in range(6)]
    cs += [k.p, k.q, k.p * 5]  # c = 0 mod p or mod q
    lines = [_sign_line(k, bm.i2osp(c, k.klen)) for c in cs]
    want = ["%d %s" % (st, s.hex()) for st, s in (bm.blind_sign(k, bm.i2osp(c, k.klen)) for c in cs)]
    # inconsistent CRT fields fail the check (at random c)
    dp, dq, qinv = k.crt()
    for crt in ((dp ^ 2, dq, qinv), (dp, dq + 2, qinv), (dp, dq, (qinv + 1) % k.p)):
        for c in cs[7:10]:
            lines.append(_sign_line(k, bm.i2osp(c, k.klen), crt))
            assert bm.blind_sign_crt(k, *crt, bm.i2osp(c, k.klen))[0] == 2
            want.append("2 " + "00" * k.klen)
    assert run(lines) == want


@pytest.mark.parametrize("name", ["rsa2048", "rsa3072", "rsa3073", "rsa2048e3", "rsa2048u", "rsa3000u", "rsa4096"])
def test_verify_failure_classes(run, name):
    k = bm.all_keys()[name]
    _, wn = _classes(k)
    rng = random.Random(name + "v")
    lines, want = [], []
    for slen in (48, 0):
        for msg in (b"", b"m" * 111, rng.randbytes(112), rng.randbytes(300)):
            for label, s, st in bm.tampered(k, slen, msg, rng):
                lines.append(f"verify {wn} {slen} {_hx(k.n)} {_hx(k.e)} {msg.hex() or '-'} {s.hex()}")
                want.append(str(st))
            # the valid signature under the other salt length
            s = bm.tampered(k, slen, msg, rng)[0][1]
            lines.append(f"verify {wn} {48 - slen} {_hx(k.n)} {_hx(k.e)} {msg.hex() or '-'} {s.hex()}")
            want.append("2")
    assert run(lines) == want
