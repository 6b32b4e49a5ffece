"""circl_b200/csrc/nistp.cuh with the P-384 and P-521 curve types, compiled for the host (g++, no GPU) through
tests/cpp/test_nistp_host.cpp, against Python integers: the field operations at 0, 1, p - 1 and random values; fixed-
and variable-base multiplication at k = 1, 2, n - 1, n - 2, at scalars whose signed radix-16 digits below the top one
are all -8, all 7, all 0 but one or a repeating -8 / 0 / 7 / -1 pattern (checked against a Python model of the
recoding), at P-521's 131st digit and at random scalars; the scalar and point checks at their edges, 66-byte P-521 rows included; and
DeriveKeyPair's range test on boundary candidates."""
import os
import random
import subprocess

import pytest

from nistp_model import CURVES, enc, mul

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("nistp") / "nistp_host")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Wno-unknown-pragmas",
                        os.path.join(ROOT, "tests", "cpp", "test_nistp_host.cpp"), "-o", path],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return path


@pytest.fixture(params=[384, 521], ids=["p384", "p521"])
def curve(request, exe):
    c = CURVES[request.param]

    def go(lines):
        out = subprocess.run([exe, str(request.param)], input="\n".join(lines) + "\n", capture_output=True, text=True,
                             timeout=600)
        assert out.returncode == 0, out.stderr
        res = out.stdout.splitlines()
        assert len(res) == len(lines)
        return res
    return c, go


def _h(c, x):
    return x.to_bytes(c.nbytes, "big").hex()


def test_field_operations(curve):
    c, run = curve
    P = c.p
    rng = random.Random(c.bits)
    vals = [0, 1, 2, P - 1, P - 2, 2**(c.bits - 1), 2**(c.bits - 2) + 1] + [rng.randrange(P) for _ in range(30)]
    lines, want = [], []
    for a in vals:
        for b in (vals[:7] + [rng.randrange(P) for _ in range(3)]):
            for op, v in (("add", (a + b) % P), ("sub", (a - b) % P), ("mul", a * b % P)):
                lines.append(f"{op} {_h(c, a)} {_h(c, b)}")
                want.append(_h(c, v))
        lines.append(f"sqr {_h(c, a)}")
        want.append(_h(c, a * a % P))
        lines.append(f"inv {_h(c, a)}")
        want.append(_h(c, pow(a, P - 2, P)))
    assert run(lines) == want


ND = {384: 96, 521: 131}  # signed radix-16 digits of a scalar


def _recode(c, k):
    """nistp.cuh's recoding in Python integers: k' (k or n - k, below 2^(bitlen(n) - 1)) plus 8 in each of the ND
    nibbles; digit i is nibble i minus 8, the top digit what is left above the lower ones, minus 8."""
    nd = ND[c.bits]
    kp = k if k < 2**(c.n.bit_length() - 1) else c.n - k
    t = kp + sum(8 * 16**i for i in range(nd))
    return [((t >> (4 * i)) & 15) - 8 for i in range(nd - 1)] + [(t >> (4 * (nd - 1))) - 8]


def _from_digits(ds):
    return sum(d * 16**i for i, d in enumerate(ds))


def _digit_scalars(c):
    """Scalars k' < 2^(bitlen(n) - 1) with chosen digits, each with n - k' (the same digits after the flip): every
    digit below the top one -8 (table entry 8, negated), 7, or 0 but one, and a repeating -8, 0, 7, -1 pattern."""
    nd = ND[c.bits]
    cases = [[-8] * (nd - 1) + [1], [7] * (nd - 1) + [0], [0] * (nd - 2) + [1, 0],
             [(-8, 0, 7, -1)[i % 4] for i in range(nd - 1)] + [1]]
    if c.bits == 384:  # a top digit of 8 (P-384's top digit is in [0, 8])
        cases.append([-8] * (nd - 1) + [8])
    ks = []
    for ds in cases:
        kp = _from_digits(ds)
        assert 0 < kp < 2**(c.n.bit_length() - 1)
        assert _recode(c, kp) == ds and _recode(c, c.n - kp) == ds
        ks += [kp, c.n - kp]
    return ks


def _scalars(c):
    N = c.n
    rng = random.Random(c.bits + 7)
    ks = [1, 2, 3, 8, 9, 16, N - 1, N - 2, N - 8, N // 2, N // 2 + 1, 2**(c.bits - 1) - 1, 2**(c.bits - 2)]
    ks += _digit_scalars(c)
    if c.bits == 521:  # nibble 129 of k' at 15: P-521's 131st digit is 1
        kp = 2**520 - 1 - 2**300
        assert _recode(c, kp)[-1] == 1
        ks += [kp, N - kp]
    return [k for k in ks if 0 < k < N] + [rng.randrange(1, N) for _ in range(12)]


def test_fixed_and_variable_base(curve):
    c, run = curve
    rng = random.Random(c.bits + 11)
    lines, want = [], []
    for k in _scalars(c):
        kp = mul(c, k, c.g)
        lines.append(f"base {_h(c, k)}")
        want.append("0 " + enc(c, kp).hex())
        pt = mul(c, rng.randrange(1, c.n), c.g)
        lines.append(f"shared {_h(c, k)} {enc(c, pt).hex()}")
        want.append("0 " + _h(c, mul(c, k, pt)[0]))
        lines.append(f"shared {_h(c, k)} {enc(c, c.g).hex()}")
        want.append("0 " + _h(c, kp[0]))
    assert run(lines) == want


def test_scalar_and_point_checks(curve):
    c, run = curve
    N, P, nb = c.n, c.p, c.nbytes
    top = 2**(8 * nb) - 1
    ks = {0: 0, 1: 1, N - 1: 1, N: 0, N + 1: 0, top: 0, 2**c.bits - 1: 0}
    if c.bits == 521:  # a leading byte of 0x02 or more is >= n; 0x01 with the rest below n is not
        ks.update({2 << (8 * (nb - 1)): 0, 0xff << (8 * (nb - 1)): 0, (1 << (8 * (nb - 1))) + 5: 1})
    lines = [f"scalar {_h(c, k)}" for k in ks]
    assert run(lines) == [str(v) for v in ks.values()]
    g = enc(c, c.g)
    x, y = c.g
    bad = {
        "off curve": b"\x04" + x.to_bytes(nb, "big") + ((y + 1) % P).to_bytes(nb, "big"),
        "X = p": b"\x04" + P.to_bytes(nb, "big") + y.to_bytes(nb, "big"),
        "Y = p": b"\x04" + x.to_bytes(nb, "big") + P.to_bytes(nb, "big"),
        "zero": bytes(c.npk),
        "zero coordinates": b"\x04" + bytes(2 * nb),
        "all ones": b"\xff" * c.npk,
    }
    if P + x < 2**(8 * nb):
        bad["X = p + x"] = b"\x04" + (P + x).to_bytes(nb, "big") + y.to_bytes(nb, "big")
    if c.bits == 521:  # bits above 521 in a coordinate row
        bad["X + 2^521"] = b"\x04" + (x + 2**521).to_bytes(nb, "big") + y.to_bytes(nb, "big")
        bad["Y + 2^527"] = b"\x04" + x.to_bytes(nb, "big") + (y + 2**527).to_bytes(nb, "big")
    for pre in (0x00, 0x02, 0x03, 0x05):
        bad[f"prefix {pre:#x}"] = bytes([pre]) + g[1:]
    good = [g, enc(c, mul(c, N - 1, c.g)), enc(c, mul(c, 2, c.g))]
    lines = [f"point {b.hex()}" for b in bad.values()] + [f"point {b.hex()}" for b in good]
    assert run(lines) == ["0"] * len(bad) + ["1"] * len(good)
    zp, zs = "00" * c.npk, "00" * nb
    lines = [f"base {_h(c, 0)}", f"base {_h(c, N)}", f"base {(b'\xff' * nb).hex()}",
             f"shared {_h(c, 5)} {bad['off curve'].hex()}", f"shared {_h(c, N)} {g.hex()}",
             f"shared {_h(c, 0)} {bad['prefix 0x2'].hex()}"]
    assert run(lines) == ["2 " + zp, "2 " + zp, "2 " + zp, "1 " + zs, "2 " + zs, "3 " + zs]


def test_candidate_range(curve):
    """DeriveKeyPair's candidate test (shortkem.go:63-90) at its boundaries, after the bitmask of byte 0."""
    c, run = curve
    N, nb = c.n, c.nbytes
    cands = [0, 1, N - 1, N, 2**(8 * nb) - 1, 2**c.bits - 1]
    if c.bits == 521:  # leading bytes 0x02..0xff are masked down to bit 0 before the test
        cands += [2 << (8 * (nb - 1)), (0xfe << (8 * (nb - 1))) + 7, (0x03 << (8 * (nb - 1))) + 7, N + (0xfe << (8 * (nb - 1)))]
    lines, want = [], []
    for v in cands:
        raw = v.to_bytes(nb, "big")
        m = bytes([raw[0] & c.mask0]) + raw[1:]
        lines.append(f"candidate {raw.hex()} {c.mask0:02x}")
        want.append(f"{int(0 < int.from_bytes(m, 'big') < N)} {m.hex()}")
    assert run(lines) == want
