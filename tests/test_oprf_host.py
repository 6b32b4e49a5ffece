"""circl_b200/csrc/oprf.cuh compiled for the host (g++, no GPU) through tests/cpp/test_oprf_host.cpp, against Python
integers and tests/oprf_model.py: scalar mul, add, sub and inversion mod n at 0, 1, n - 1 and random values; the wide
reduction of hash_to_field strings at the largest inputs; decompression at both parities, X = p - 1, X >= p and
non-residues; expand_message_xmd and hash_to_curve (u, Q0, Q1, P) against the RFC 9380 vectors; and DeriveKey,
Evaluate (with the proof) and FullEvaluate against every NIST-suite RFC 9497 vector and the model."""
import os
import random
import subprocess

import pytest

import oprf_model as om
from conftest import load_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BITS = {"P256-SHA256": 256, "P384-SHA384": 384, "P521-SHA512": 521}


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("oprf") / "oprf_host")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Wno-unknown-pragmas",
                        os.path.join(ROOT, "tests", "cpp", "test_oprf_host.cpp"), "-o", path],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return path


@pytest.fixture(params=list(BITS), ids=["p256", "p384", "p521"])
def suite(request, exe):
    s = om.SUITES[request.param]

    def go(lines):
        out = subprocess.run([exe, str(BITS[request.param])], input="\n".join(lines) + "\n", capture_output=True,
                             text=True, timeout=600)
        assert out.returncode == 0, out.stderr
        res = out.stdout.splitlines()
        assert len(res) == len(lines)
        return res
    return s, go


def _h(s, x):
    return x.to_bytes(s.nbytes, "big").hex()


def _x(b):
    return b.hex() if b else "-"


def test_scalar_arithmetic(suite):
    s, run = suite
    N = s.n
    rng = random.Random(s.bits)
    vals = [0, 1, 2, N - 1, N - 2, N // 2] + [rng.randrange(N) for _ in range(20)]
    lines, want = [], []
    for a in vals:
        for b in vals[:6] + [rng.randrange(N) for _ in range(3)]:
            for op, v in (("scmul", a * b % N), ("scadd", (a + b) % N), ("scsub", (a - b) % N)):
                lines.append(f"{op} {_h(s, a)} {_h(s, b)}")
                want.append(_h(s, v))
        lines.append(f"scinv {_h(s, a)}")
        want.append(_h(s, pow(a, N - 2, N)))
    assert run(lines) == want


def test_wide_reduction(suite):
    s, run = suite
    rng = random.Random(s.bits + 1)
    vals = [0, 1, s.n, s.p, 2**(8 * s.L) - 1, 2**(8 * s.L) - 2, s.n * (2**(8 * s.L) // s.n)] + \
        [rng.randrange(2**(8 * s.L)) for _ in range(20)]
    lines, want = [], []
    for v in vals:
        b = v.to_bytes(s.L, "big").hex()
        lines += [f"widen {b}", f"widep {b}"]
        want += [_h(s, v % s.n), _h(s, v % s.p)]
    assert run(lines) == want


def test_decompression(suite):
    s, run = suite
    rng = random.Random(s.bits + 2)
    pts = [s.g, om.mul(s, s.n - 1, s.g)] + [om.mul(s, rng.randrange(1, s.n), s.g) for _ in range(10)]
    rows = [om.compress(s, p) for p in pts]
    assert {r[0] for r in rows} == {2, 3}
    want = ["1 " + _h(s, x) + " " + _h(s, y) for x, y in pts]
    x = s.p - 1
    rhs = (x ** 3 - 3 * x + s.b) % s.p
    bad = [b"\x04" + r[1:] for r in rows[:2]] + [b"\x00" + rows[0][1:], bytes([rows[0][0] | 4]) + rows[0][1:]]
    bad += [b"\x02" + s.p.to_bytes(s.nbytes, "big"), b"\x03" + (2**(8 * s.nbytes) - 1).to_bytes(s.nbytes, "big")]
    nonres = [v for v in range(1, 200) if not om._is_square(s, (v ** 3 - 3 * v + s.b) % s.p)][:3]
    bad += [b"\x02" + v.to_bytes(s.nbytes, "big") for v in nonres]
    lines = [f"decode {r.hex()}" for r in rows] + [f"decode 02{_h(s, x)}"] + [f"decode {b.hex()}" for b in bad]
    res = run(lines)
    assert res[:len(rows)] == want
    pm1 = om.decompress(s, bytes.fromhex("02" + _h(s, x)))
    assert res[len(rows)] == ("1 " + _h(s, pm1[0]) + " " + _h(s, pm1[1]) if pm1 else "0")
    assert (pm1 is not None) == om._is_square(s, rhs)
    assert res[len(rows) + 1:] == ["0"] * len(bad)


XMD = {256: ["expand_message_xmd_SHA256_38.json.gz"], 384: [], 521: ["expand_message_xmd_SHA512_38.json.gz"]}


def test_expand_message_xmd(suite):
    s, run = suite
    lines, want = [], []
    for name in XMD[s.bits]:
        f = load_golden(name)
        for v in f["tests"]:
            n = int(v["len_in_bytes"], 16)
            if n <= 2 * s.L:
                lines.append(f"xmd {n} {f['DST'].encode().hex()} {_x(v['msg'].encode())}")
                want.append(v["uniform_bytes"])
    # the suite's own hash with the OPRF DSTs, against the model
    for msg in (b"", b"abc", bytes(range(200))):
        for n in (s.L, 2 * s.L):
            dst = b"HashToGroup-" + om.context(s, 2)
            lines.append(f"xmd {n} {dst.hex()} {_x(msg)}")
            want.append(om.expand_message_xmd(s.hash, msg, dst, n).hex())
    assert run(lines) == want


H2C = {256: "h2c_P256_XMD-SHA-256_SSWU_RO_.json.gz", 384: "h2c_P384_XMD-SHA-384_SSWU_RO_.json.gz",
       521: "h2c_P521_XMD-SHA-512_SSWU_RO_.json.gz"}


def test_hash_to_curve(suite):
    s, run = suite
    f = load_golden(H2C[s.bits])
    lines, want = [], []
    for v in f["vectors"]:
        lines.append(f"h2c {f['dst'].encode().hex()} {_x(v['msg'].encode())}")
        want.append(" ".join([_h(s, int(u, 16)) for u in v["u"]] +
                             [_h(s, int(v[q][c], 16)) for q in ("Q0", "Q1", "P") for c in ("x", "y")]))
    assert run(lines) == want


def test_rfc9497_vectors(suite):
    s, run = suite
    lines, want = [], []
    for tv in load_golden("oprf_rfc9497.json.gz"):
        if tv["identifier"] != s.identifier:
            continue
        mode = tv["mode"]
        lines.append(f"derive {mode} {tv['seed']} {tv['keyInfo']}")
        want.append(tv["skSm"] + " " + om.derive_key(s, mode, bytes.fromhex(tv["seed"]),
                                                      bytes.fromhex(tv["keyInfo"]))[1].hex())
        for v in tv["vectors"]:
            info = v.get("Info", "") or "-"
            r = v["Proof"]["r"] if "Proof" in v else "-"
            lines.append(f"evaluate {mode} {tv['skSm']} {r} {info} {' '.join(v['BlindedElement'].split(','))}")
            want.append("0 " + " ".join(v["EvaluationElement"].split(",")) + " " +
                        (v["Proof"]["proof"] if "Proof" in v else "-"))
            for inp, out in zip(v["Input"].split(","), v["Output"].split(",")):
                lines.append(f"full {mode} {tv['skSm']} {info} {inp}")
                want.append("0 " + out)
    assert run(lines) == want


def test_model_parity_and_failures(suite):
    """Random keys, inputs, r and info against the model, m = 3, and each status bit."""
    s, run = suite
    rng = random.Random(s.bits + 3)
    lines, want = [], []
    for mode in (0, 1, 2):
        sk = om.i2osp(rng.randrange(1, s.n), s.Ns)
        r = om.i2osp(rng.randrange(1, s.n), s.Ns)
        info = bytes(rng.randrange(256) for _ in range(rng.randrange(0, 300)))
        inp = bytes(rng.randrange(256) for _ in range(rng.randrange(0, 300)))
        bl = [om.compress(s, om.mul(s, rng.randrange(1, s.n), s.g)) for _ in range(3)]
        ev, proof = om.evaluate(s, mode, sk, bl, r if mode else None, info)
        lines.append(f"evaluate {mode} {sk.hex()} {r.hex()} {_x(info)} {' '.join(b.hex() for b in bl)}")
        want.append("0 " + " ".join(e.hex() for e in ev) + " " + (proof.hex() if proof else "-"))
        lines.append(f"full {mode} {sk.hex()} {_x(info)} {_x(inp)}")
        want.append("0 " + om.full_evaluate(s, mode, sk, inp, info).hex())
    assert run(lines) == want
    # status bits: an element off the curve (1), sk = 0 (2), r = n (4), t = 0 (8)
    g = om.compress(s, s.g)
    sk = om.i2osp(5, s.Ns)
    x = next(v for v in range(1, 200) if not om._is_square(s, (v ** 3 - 3 * v + s.b) % s.p))
    offc = b"\x02" + x.to_bytes(s.nbytes, "big")
    tz = om.i2osp(s.n - om.info_scalar(s, b"i"), s.Ns)
    res = run([f"evaluate 1 {sk.hex()} {_h(s, 1)} - {g.hex()} {offc.hex()}",
               f"evaluate 1 {_h(s, 0)} {_h(s, 1)} - {g.hex()}",
               f"evaluate 1 {sk.hex()} {_h(s, s.n)} - {g.hex()}",
               f"evaluate 2 {tz.hex()} {_h(s, 1)} {b'i'.hex()} {g.hex()}",
               f"full 2 {tz.hex()} {b'i'.hex()} 00",
               f"full 0 {_h(s, s.n)} - 00"])
    assert [int(l.split()[0]) for l in res] == [1, 2, 4, 8, 8, 2]
