"""The partially blind RSA code of circl_b200/csrc/rsa.cuh compiled for the host (g++, no GPU) through
tests/cpp/test_pbrsa_host.cpp, against tests/pbrsa_model.py and Python integers: e' on every fixture key, the windowed
public exponentiation at 32 to 128 words, the Fermat inverse mod p' with its odd lift, the Miller-Rabin test, and
whole BlindSign and Verify (the unbalanced key included)."""
import os
import random
import subprocess

import pytest

import brsa_model as bm
import pbrsa_model as pm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = ["strong2048", "safe3072", "safe4096", "safe2050", "safe2052", "safe3073", "safe2048u"]
METAS = [b"", b"\x00", b"metadata", bytes(range(120)), bytes(124), bytes(range(256)) * 4 + b"x"]


@pytest.fixture(scope="module")
def run(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("pbrsa") / "pbrsa_host")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Wno-unknown-pragmas",
                        os.path.join(ROOT, "tests", "cpp", "test_pbrsa_host.cpp"), "-o", path],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]

    def go(lines):
        out = subprocess.run([path], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=900)
        assert out.returncode == 0, out.stderr
        res = out.stdout.splitlines()
        assert len(res) == len(lines)
        return res
    return go


def _h(x, w):
    return x.to_bytes(4 * w, "big").hex()


def _hx(x):
    return x.to_bytes((x.bit_length() + 7) // 8 or 1, "big").hex()


def _classes(k):
    wp = next(w for w in (32, 48, 64) if max(k.p.bit_length(), k.q.bit_length()) <= 32 * w)
    wn = next(w for w in (64, 96, 128) if k.n.bit_length() <= 32 * w)
    return wp, wn


@pytest.mark.parametrize("name", KEYS)
def test_derived_exponent(run, name):
    k = pm.keys()[name]
    _, wn = _classes(k)
    lines = [f"derive {wn} {_hx(k.n)} {m.hex() or '-'}" for m in METAS]
    assert run(lines) == [_h(pm.derive_public_key(k.n, m), wn // 2) for m in METAS]


@pytest.mark.parametrize("w", [32, 48, 64, 96, 128])
def test_public_exponentiation(run, w):
    rng = random.Random(w)
    lines, want = [], []
    for top in (0xffffffff, 0x80000000, 0x3):
        m = (top << (32 * w - 32)) | rng.getrandbits(32 * w - 32) | 1
        for bits in (1, 5, 6, 31, 32, 33, 16 * w - 2, 16 * w):
            for e in {1, (1 << bits) - 1, rng.getrandbits(bits) | 1, 1 << (bits - 1)}:
                for x in (0, 1, m - 1, rng.randrange(m)):
                    lines.append(f"expw {w} {_h(m, w)} {_h(x, w)} {_h(e, w)} {bits}")
                    want.append(_h(pow(x, e, m), w))
    assert run(lines) == want


@pytest.mark.parametrize("name", KEYS)
def test_inverse_and_lift(run, name):
    k = pm.keys()[name]
    wp, _ = _classes(k)
    rng = random.Random(name + "h")
    lines, want = [], []
    for p in (k.p, k.q):
        es = [pm.derive_public_key(k.n, m) for m in METAS] + [3, 5, (p - 1) // 2 + 2, (p - 1) // 2 - 2]
        for e in es:
            e |= 1
            if e % ((p - 1) // 2) == 0:
                continue
            d = pow(e, -1, p - 1)
            for c in (0, 1, p - 1, rng.randrange(p)):
                lines.append(f"half {wp} {_hx(p)} {_h(e % (1 << (32 * wp)), wp)} {_h(c, wp)}")
                want.append(_h(pow(c, d, p), wp))
    # both parities of e'^-1 mod p' occur
    ph = (k.p - 1) // 2
    assert {pow(pm.derive_public_key(k.n, m) % ph, -1, ph) % 2 for m in METAS} == {0, 1}
    assert run(lines) == want


def test_miller_rabin(run):
    ks = pm.keys()
    lines, want = [], []
    for name, k in ks.items():
        for p in (k.p, k.q):
            w = next(w for w in (32, 48, 64) if p.bit_length() <= 32 * w)
            lines += [f"prime {w} {_hx((p - 1) // 2)}", f"prime {w} {_hx(p)}", f"prime {w} {_hx(p * 3 // 4 * 2 + 1)}"]
            want += ["1", "1", "0"]
    u = bm.all_keys()["rsa2048u"]  # primes = 3 mod 4 whose halves are composite
    for p in (u.p, u.q):
        w = next(w for w in (32, 48, 64) if p.bit_length() <= 32 * w)
        lines.append(f"prime {w} {_hx((p - 1) // 2)}")
        want.append("0")
    lines += ["prime 32 03", "prime 32 05", "prime 32 07", "prime 32 09", "prime 32 " + _hx(561), "prime 32 " +
              _hx(3215031751)]  # 561 and 3215031751 are Carmichael / strong pseudoprimes to small bases
    want += ["1", "1", "1", "0", "0", "0"]
    assert run(lines) == want


def _sign_line(k, meta, c, qinv=None):
    wp, wn = _classes(k)
    qinv = pow(k.q, -1, k.p) if qinv is None else qinv
    return f"sign {wp} {wn} {_hx(k.n)} {_hx(k.p)} {_hx(k.q)} {_hx(qinv)} {meta.hex() or '-'} {c.hex()}"


@pytest.mark.parametrize("name", KEYS)
def test_blind_sign(run, name):
    k = pm.keys()[name]
    rng = random.Random(name + "s")
    lines, want = [], []
    for i, meta in enumerate(METAS):
        cs = [rng.randrange(k.n) for _ in range(2)]
        if i == 0:
            cs += [0, 1, k.n - 1, k.n, k.n + 1, (1 << (8 * k.klen)) - 1, k.p, k.q * 3]
        for c in cs:
            cb = bm.i2osp(c, k.klen)
            lines.append(_sign_line(k, meta, cb))
            st, s = pm.blind_sign(k, cb, meta)
            want.append(f"{st} {s.hex()}")
    # a wrong qinv fails the check
    c = bm.i2osp(rng.randrange(k.n), k.klen)
    lines.append(_sign_line(k, b"m", c, (pow(k.q, -1, k.p) + 1) % k.p))
    want.append("2 " + "00" * k.klen)
    assert run(lines) == want


@pytest.mark.parametrize("name", KEYS)
def test_verify(run, name):
    k = pm.keys()[name]
    _, wn = _classes(k)
    rng = random.Random(name + "v")
    lines, want = [], []
    for meta in METAS:
        msg = rng.randbytes(rng.randrange(0, 300))
        sig = pm.sign(k, msg, meta, rng)
        other = meta + b"!" if meta else b"!"
        bad = bytearray(sig)
        bad[-1] ^= 1
        for mt, m, s in ((meta, msg, sig), (other, msg, sig), (meta, msg + b"x", sig), (meta, msg, bytes(bad)),
                         (meta, msg, bm.i2osp(k.n, k.klen)), (meta, msg, bm.i2osp(k.n + 1, k.klen))):
            lines.append(f"verify {wn} {_hx(k.n)} {mt.hex() or '-'} {m.hex() or '-'} {s.hex()}")
            want.append(str(pm.verify_status(k, m, mt, s)))
    assert want.count("0") == len(METAS) and want.count("1") == 2 * len(METAS)
    assert run(lines) == want
