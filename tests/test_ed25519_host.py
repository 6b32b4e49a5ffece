"""circl_b200/csrc/ed25519.cuh compiled for the host (g++, no GPU) through tests/cpp/test_ed25519_host.cpp: SHA-512
against hashlib, scalars mod L against Python integers, point decoding edge cases, keygen / sign / verify against
OpenSSL's Ed25519 (the `cryptography` package) and the reference's RFC 8032 and Wycheproof vectors, and decoding, the
double multiplication and verify on small-order and mixed-order keys and non-canonical encodings against the
Python-integer model (tests/ed25519_model.py)."""
import hashlib
import os
import random
import subprocess

import pytest

import ed25519_model as M
from conftest import load_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 2**255 - 19
L = 2**252 + 27742317777372353535851937790883648493


@pytest.fixture(scope="module")
def run(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("ed25519") / "ed25519_host")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", os.path.join(ROOT, "tests", "cpp", "test_ed25519_host.cpp"),
                        "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]

    def go(lines):
        out = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stderr
        res = out.stdout.splitlines()
        assert len(res) == len(lines)
        return res
    return go


def _le(v, n=32):
    return (v % 2**(8 * n)).to_bytes(n, "little").hex()


def _h(m):
    return m.hex() if m else "-"


def test_sha512_block_boundaries(run):
    rng = random.Random(1)
    lens = [32, 33, 63, 64, 65, 111, 112, 113, 127, 128, 129, 239, 240, 241, 255, 256, 1000, 10000]
    msgs = [bytes(rng.randrange(256) for _ in range(n)) for n in lens]
    got = run(["sha512 " + m.hex() for m in msgs])
    assert got == [hashlib.sha512(m).hexdigest() for m in msgs]


def test_reduce_mod_order(run):
    rng = random.Random(2)
    xs = [0, 1, L - 1, L, L + 1, 2 * L, 3 * L - 1, 2**252, 2**256 - 1, 2**512 - 1, (2**512 // L) * L, (2**512 // L) * L - 1]
    xs += [rng.getrandbits(512) for _ in range(300)] + [rng.getrandbits(300) for _ in range(50)]
    got = run(["reduce " + _le(x, 64) for x in xs])
    assert got == [_le(x % L) for x in xs]


def test_calculate_s(run):
    rng = random.Random(3)
    cases = [(0, 0, 0), (L - 1, L - 1, 2**256 - 1), (L - 1, 1, 1), (0, L - 1, 2**255 - 8), (1, 0, 2**254)]
    for _ in range(300):
        a = rng.getrandbits(256)
        a = (a & ~7 & (2**255 - 1)) | 2**254  # clamped
        cases.append((rng.randrange(L), rng.randrange(L), a))
    got = run(["muladd %s %s %s" % (_le(r), _le(k), _le(a)) for r, k, a in cases])
    assert got == [_le((r + k * a) % L) for r, k, a in cases]
    ss = [0, L - 1, L, L + 1, 2**256 - 1, 2**253]
    assert run(["canon " + _le(s) for s in ss]) == ["1" if s < L else "0" for s in ss]


def test_decode_edge_cases(run):
    rng = random.Random(4)
    ys = [(0, 0), (1, 0), (1, 1), (P - 1, 0), (P - 1, 1), (P, 0), (P + 1, 0), (2**255 - 1, 0), (2**255 - 1, 1), (2, 0)]
    ys += [(rng.randrange(P), rng.getrandbits(1)) for _ in range(200)]
    got = run(["decode " + _le(y | (s << 255)) for y, s in ys])
    n_bad = 0
    for (y, s), g in zip(ys, got):
        pt = M.decode(bytes.fromhex(_le(y | (s << 255))))
        if pt is None:
            assert g == "0", (y, s)
            n_bad += 1
        else:
            assert g == "1" + M.encode(pt).hex(), (y, s)
    assert 50 < n_bad < 190  # about half of the random y have no square root


def test_keygen_sign_verify_against_openssl(run):
    from cryptography.hazmat.primitives.asymmetric.ed25519 import Ed25519PrivateKey
    rng = random.Random(5)
    lens = [0, 1, 111, 112, 127, 128, 239, 240, 10000]
    lines, exp = [], []
    for i in range(40):
        seed = bytes(rng.randrange(256) for _ in range(32))
        sk = Ed25519PrivateKey.from_private_bytes(seed)
        A = sk.public_key().public_bytes_raw()
        msg = bytes(rng.randrange(256) for _ in range(lens[i % len(lens)]))
        sig = sk.sign(msg)
        bad = bytearray(sig)
        bad[rng.randrange(64)] ^= 1 << rng.randrange(8)
        lines += ["keygen " + seed.hex(), "sign %s %s %s" % (seed.hex(), A.hex(), _h(msg)),
                  "verify %s %s %s" % (A.hex(), _h(msg), sig.hex()), "verify %s %s %s" % (A.hex(), _h(msg), bytes(bad).hex())]
        exp += [A.hex(), sig.hex(), "1", "0"]
    assert run(lines) == exp


def test_fixed_base_and_double_mult(run):
    """[k]B for any k < 2^255 equals [k mod L]B, and encode([s]B + [k]A) for A = [a]B equals encode([(s + k a) mod L]B)."""
    from cryptography.hazmat.primitives.asymmetric.ed25519 import Ed25519PrivateKey
    rng = random.Random(6)
    cases = [(rng.getrandbits(255), rng.getrandbits(255), rng.randrange(2**253)) for _ in range(30)]
    cases += [(2**255 - 1, L - 1, L - 1), (L, 0, 1), (0, 1, 0)]
    got = run(["base " + _le(a) for a, _, _ in cases] + ["base " + _le(a % L) for a, _, _ in cases])
    As = got[:len(cases)]
    assert As == got[len(cases):]
    dm = run(["dmul %s %s %s" % (_le(s), _le(k), A) for (a, s, k), A in zip(cases, As)])
    assert dm == run(["base " + _le((s + k * a) % L) for a, s, k in cases])
    seed = bytes(range(32))
    assert run(["keygen " + seed.hex()])[0] == Ed25519PrivateKey.from_private_bytes(seed).public_key().public_bytes_raw().hex()


def test_x25519_keygen_through_refactored_core(run):
    rng = random.Random(7)
    ks = [bytes(rng.randrange(256) for _ in range(32)) for _ in range(50)] + [bytes(32), b"\xff" * 32]
    for line in run(["x25519 " + k.hex() for k in ks]):
        u1, u2 = line.split()
        assert u1 == u2


def test_rfc8032_and_wycheproof_vectors(run):
    v = load_golden("ed25519_vectors.json.gz")
    lines, exp = [], []
    for t in v["rfc8032"] + v["sign_input"][:256]:
        seed, A, msg, sig = (bytes.fromhex(t[k]) for k in ("seed", "pk", "msg", "sig"))
        lines += ["keygen " + seed.hex(), "sign %s %s %s" % (seed.hex(), A.hex(), _h(msg)),
                  "verify %s %s %s" % (A.hex(), _h(msg), sig.hex())]
        exp += [A.hex(), sig.hex(), "1"]
    for t in v["wycheproof"]:
        if len(bytes.fromhex(t["sig"])) != 64:
            continue  # the wrong-length signatures are rejected before any arithmetic
        lines.append("verify %s %s %s" % (t["pk"], _h(bytes.fromhex(t["msg"])), t["sig"]))
        exp.append("1" if t["valid"] else "0")
    assert run(lines) == exp


def test_decode_torsion_and_non_canonical_encodings(run):
    """The 8 points of order dividing 8 decode to themselves; the 38 encodings with y >= p, and x = 0 with the sign
    bit (y = 1, y = p - 1), are rejected."""
    tors = [M.encode(T) for T in M.TORSION]
    assert run(["decode " + e.hex() for e in tors]) == ["1" + e.hex() for e in tors]
    bad = [y | s << 255 for y in range(P, 2**255) for s in (0, 1)] + [1 | 1 << 255, P - 1 | 1 << 255]
    assert len(bad) == 40 and all(M.decode(bytes.fromhex(_le(v))) is None for v in bad)
    assert run(["decode " + _le(v) for v in bad]) == ["0"] * 40


def test_double_mult_small_order_points(run):
    """encode([s] B + [k] T) for every T of order dividing 8, at k around multiples of 8 and at random k, where the
    table of the multiples 1..8 T passes through the identity."""
    rng = random.Random(8)
    ks = [0, 1, 2, 3, 4, 7, 8, 9, 15, 16, 17, L - 1, 2**252] + [rng.randrange(L) for _ in range(4)]
    cases = [(rng.randrange(L), k, j) for j in range(8) for k in ks]
    got = run(["dmul %s %s %s" % (_le(s), _le(k), M.encode(M.TORSION[j]).hex()) for s, k, j in cases])
    sB = {s: M.mul(s, M.B) for s, _, _ in cases}
    assert got == [M.encode(M.add(sB[s], M.TORSION[(k * j) % 8])).hex() for s, k, j in cases]


def test_torsion_cases_against_model(run):
    """verify gives the model's verdict on every small-order, mixed-order and non-canonical case."""
    cases = M.torsion_cases()
    got = run(["verify %s %s %s" % (pk.hex(), _h(msg), sig.hex()) for _, pk, msg, sig, _ in cases])
    assert got == ["1" if c[4] else "0" for c in cases], [c[0] for c, g in zip(cases, got) if g != ("1" if c[4] else "0")]
