"""circl_b200/csrc/ed448.cuh compiled for the host (g++, no GPU) through tests/cpp/test_ed448_host.cpp: SHAKE256 over
the three segments against hashlib, scalars mod l against Python integers, the group-law formulas at the accumulator
bound, point decoding edge cases, the fixed base, and keygen / sign / verify against the oracle, OpenSSL's Ed448 and
the Python model of the reference's verification equation (tests/ed448_model.py)."""
import hashlib
import os
import random
import subprocess

import pytest

import ed448_model as M
from conftest import load_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P, L = M.P, M.L


@pytest.fixture(scope="module")
def run(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("ed448") / "ed448_host")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", os.path.join(ROOT, "tests", "cpp", "test_ed448_host.cpp"),
                        "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]

    def go(lines):
        out = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=900)
        assert out.returncode == 0, out.stderr
        res = out.stdout.splitlines()
        assert len(res) == len(lines)
        return res
    return go


def _le(v, n=56):
    return (v % 2**(8 * n)).to_bytes(n, "little").hex()


def _h(m):
    return m.hex() if m else "-"


def test_shake_segments(run):
    rng = random.Random(1)
    cases = []
    for lc in (None, 0, 1, 127, 255):
        for npre in (0, 57, 114):
            for n in (0, 1, 7, 8, 9, 135, 136, 137, 300):
                if rng.random() < 0.5:
                    continue
                cases.append((None if lc is None else bytes(rng.randrange(256) for _ in range(lc)),)
                             + tuple(bytes(rng.randrange(256) for _ in range(k)) for k in (npre, n)))
    got = run(["shake %s %s %s" % ("none" if a is None else _h(a), _h(b), _h(c)) for a, b, c in cases])
    assert got == [hashlib.shake_256((b"" if a is None else M.dom(a)) + b + c).digest(114).hex() for a, b, c in cases]


def test_reduce_mod_order(run):
    rng = random.Random(2)
    xs = [0, 1, L - 1, L, L + 1, 4 * L, 4 * L + 3, 2**446, 2**448 - 1, 2**912 - 1, (2**912 // L) * L, (2**912 // L) * L - 1]
    xs += [rng.getrandbits(912) for _ in range(300)] + [rng.getrandbits(450) for _ in range(50)]
    assert run(["reduce " + _le(x, 114) for x in xs]) == [_le(x % L) for x in xs]


def test_muladd_and_canonical(run):
    rng = random.Random(3)
    cases = [(0, 0, 0), (L - 1, L - 1, L - 1), (L - 1, 1, 0), (1, L - 1, L - 1)]
    cases += [(rng.randrange(L), rng.randrange(L), rng.randrange(L)) for _ in range(300)]
    got = run(["muladd %s %s %s" % (_le(k), _le(s), _le(r)) for k, s, r in cases])
    assert got == [_le((k * s + r) % L) for k, s, r in cases]
    ss = [0, L - 1, L, L + 1, 2**448 - 1, 2**446, 2**448, 2**455]
    assert run(["canon " + _le(s, 57) for s in ss]) == ["1" if s < L else "0" for s in ss]


def _limbs(vals):
    return b"".join(int(v).to_bytes(4, "little", signed=True) for v in vals)


def _val(vals):
    return sum(v << (28 * i) for i, v in enumerate(vals)) % P


def test_group_law_at_the_accumulator_bound(run):
    """Every operand at the carried extreme: limbs of magnitude 2^27 (2^27 + 2^8 on limbs 1 and 9, the carry spill),
    in all-equal and alternating signs.  The results must match the formulas evaluated on the same field values."""
    top = [2**27 + (2**8 if i in (1, 9) else 0) for i in range(16)]
    pats = [top, [-v for v in top], [v if i % 2 else -v for i, v in enumerate(top)], [-v if i % 2 else v for i, v in enumerate(top)]]
    rng = random.Random(4)
    lines, exp = [], []
    for _ in range(24):
        fs = [rng.choice(pats) for _ in range(8)]
        X1, Y1, Z1, T1, X2, Y2, Z2, T2 = (_val(f) for f in fs)
        # madd: q = (x, y, dxy)
        A, B, C, Dd = X1 * X2, Y1 * Y2, T1 * Z2, Z1
        E = (X1 + Y1) * (X2 + Y2) - A - B
        F, Gg, H = Dd - C, Dd + C, B - A
        lines.append("madd " + (_limbs(sum(fs[:4], [])) + _limbs(sum(fs[4:7], []))).hex())
        exp.append(" ".join(_le(v % P) for v in (E * F, Gg * H, F * Gg, E * H)))
        # add: q = (X, Y, Z, dT)
        A, B, C, Dd = X1 * X2, Y1 * Y2, T1 * T2, Z1 * Z2
        E = (X1 + Y1) * (X2 + Y2) - A - B
        F, Gg, H = Dd - C, Dd + C, B - A
        lines.append("add " + _limbs(sum(fs, [])).hex())
        exp.append(" ".join(_le(v % P) for v in (E * F, Gg * H, F * Gg, E * H)))
        # dbl
        A, B, C = X1 * X1, Y1 * Y1, 2 * Z1 * Z1
        E = (X1 + Y1) ** 2 - A - B
        Gg, H = A + B, A - B
        F = Gg - C
        lines.append("dbl " + _limbs(sum(fs[:4], [])).hex())
        exp.append(" ".join(_le(v % P) for v in (E * F, Gg * H, F * Gg, E * H)))
    assert run(lines) == exp


def _enc(y, top):
    return _le(y) + "%02x" % top


def test_decode_edge_cases(run):
    rng = random.Random(5)
    encs = [_enc(1, 0), _enc(1, 0x80), _enc(P - 1, 0), _enc(P - 1, 0x80), _enc(0, 0), _enc(0, 0x80),
            _enc(P, 0), _enc(P + 1, 0), _enc(2**448 - 1, 0), _enc(1, 0x01), _enc(1, 0x7f), M.encode(M.G).hex(),
            (M.encode(M.G)[:56] + b"\x81").hex()]
    encs += [_enc(rng.randrange(P), rng.choice((0, 0x80))) for _ in range(150)]
    got = run(["decode " + e for e in encs])
    n_bad = 0
    for e, g in zip(encs, got):
        pt = M.decode(bytes.fromhex(e))
        if pt is None:
            assert g == "0", e
            n_bad += 1
        else:
            assert g == "1" + M.encode(pt).hex(), e
    assert 40 < n_bad < 140


def test_fixed_base(run):
    from oracle import ed448 as oe
    rng = random.Random(6)
    ks = [0, 1, 2, L - 1, 2**446 - 1] + [rng.randrange(L) for _ in range(20)] + [rng.getrandbits(447) for _ in range(10)]
    assert run(["base " + _le(k) for k in ks]) == [M.encode(M.mul(k, M.G)).hex() for k in ks]
    clamped = [2**447, 2**448 - 4, L, 2**447 + 2**446]
    assert run(["basered " + _le(k) for k in clamped]) == [M.encode(M.mul(k % L, M.G)).hex() for k in clamped]
    assert [oe.base_mult(k % L) for k in clamped] == [M.encode(M.mul(k % L, M.G)) for k in clamped]


def test_double_mult(run):
    rng = random.Random(7)
    lines, exp = [], []
    for i in range(12):
        a, s, k = rng.randrange(L), rng.randrange(L), rng.randrange(2**448)
        A = M.mul(a, M.G)
        if i % 3 == 1:
            A = M.add(A, M.TORSION[1 + i % 3])
        lines.append("dmul %s %s %s" % (_le(s), _le(k), M.encode(A).hex()))
        exp.append(M.encode(M.add(M.mul(s, M.G), M.mul(k, A))).hex())
    assert run(lines) == exp


def test_keygen_sign_verify_against_oracle_and_openssl(run):
    from cryptography.hazmat.primitives.asymmetric.ed448 import Ed448PrivateKey
    from oracle import ed448 as oe
    rng = random.Random(8)
    lens = [0, 1, 3, 25, 26, 33, 69, 70, 79, 80, 135, 136, 137, 400]
    ctxs = [b"", b"", b"c", bytes(range(255))]
    lines, exp = [], []
    for i in range(300):
        seed = bytes(rng.randrange(256) for _ in range(57))
        msg = bytes(rng.randrange(256) for _ in range(lens[i % len(lens)]))
        ctx = ctxs[i % 4]
        A, sk = oe.ed448_keygen(seed)
        sig = oe.ed448_sign(sk, msg, ctx)
        if not ctx and i % 8 == 0:
            okey = Ed448PrivateKey.from_private_bytes(seed)
            assert A == okey.public_key().public_bytes_raw() and sig == okey.sign(msg)
        bad = bytearray(sig)
        bad[rng.randrange(114)] ^= 1 << rng.randrange(8)
        lines += ["keygen " + seed.hex(), "sign %s %s %s %s" % (seed.hex(), A.hex(), _h(ctx), _h(msg)),
                  "verify %s %s %s %s" % (A.hex(), _h(ctx), _h(msg), sig.hex()),
                  "verify %s %s %s %s" % (A.hex(), _h(ctx), _h(msg), bytes(bad).hex())]
        exp += [A.hex(), sig.hex(), "1", "1" if oe.ed448_verify(A, msg, bytes(bad), ctx) else "0"]
    assert run(lines) == exp


def test_rfc8032_and_wycheproof_vectors(run):
    v = load_golden("ed448_vectors.json.gz")
    lines, exp = [], []
    for t in v["rfc8032"]:
        lines += ["keygen " + t["seed"], "sign %s %s %s %s" % (t["seed"], t["pk"], t["ctx"] or "-", t["msg"] or "-"),
                  "verify %s %s %s %s" % (t["pk"], t["ctx"] or "-", t["msg"] or "-", t["sig"])]
        exp += [t["pk"], t["sig"], "1"]
    for t in v["wycheproof"]:
        if len(t["sig"]) != 228 or len(t["pk"]) != 114:
            continue  # wrong lengths are rejected before any arithmetic
        lines.append("verify %s - %s %s" % (t["pk"], t["msg"] or "-", t["sig"]))
        exp.append("1" if t["valid"] else "0")
    assert run(lines) == exp
