"""circl_b200/csrc/p256.cuh compiled for the host (g++, no GPU) through tests/cpp/test_p256_host.cpp, against Python
integers: the field operations at 0, 1, p - 1 and random values; fixed- and variable-base multiplication at
k = 1, 2, n - 1, n - 2, at scalars whose signed radix-16 digits are all +8 or -8 and at random scalars; the scalar
and point checks at their edges."""
import os
import random
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 2**256 - 2**224 + 2**192 + 2**96 - 1
N = 0xffffffff00000000ffffffffffffffffbce6faada7179e84f3b9cac2fc632551
B = 0x5ac635d8aa3a93e7b3ebbd55769886bc651d06b0cc53b0f63bce3c3e27d2604b
G = (0x6b17d1f2e12c4247f8bce6e563a440f277037d812deb33a0f4a13945d898c296,
     0x4fe342e2fe1a7f9b8ee7eb4a7c0f9e162bce33576b315ececbb6406837bf51f5)


def _add(a, b):
    if a is None:
        return b
    if b is None:
        return a
    if a[0] == b[0]:
        if (a[1] + b[1]) % P == 0:
            return None
        lam = (3 * a[0] * a[0] - 3) * pow(2 * a[1], -1, P) % P
    else:
        lam = (b[1] - a[1]) * pow(b[0] - a[0], -1, P) % P
    x = (lam * lam - a[0] - b[0]) % P
    return x, (lam * (a[0] - x) - a[1]) % P


def mul(k, pt):
    r = None
    for bit in bin(k)[2:]:
        r = _add(r, r)
        if bit == "1":
            r = _add(r, pt)
    return r


def enc(pt):
    return b"\x04" + pt[0].to_bytes(32, "big") + pt[1].to_bytes(32, "big")


@pytest.fixture(scope="module")
def run(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("p256") / "p256_host")
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Wno-unknown-pragmas",
                        os.path.join(ROOT, "tests", "cpp", "test_p256_host.cpp"), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]

    def go(lines):
        out = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stderr
        res = out.stdout.splitlines()
        assert len(res) == len(lines)
        return res
    return go


def _h(x):
    return x.to_bytes(32, "big").hex()


def test_field_operations(run):
    rng = random.Random(256)
    vals = [0, 1, 2, P - 1, P - 2, 2**255, 2**224] + [rng.randrange(P) for _ in range(40)]
    lines, want = [], []
    for a in vals:
        for b in (vals[:7] + [rng.randrange(P) for _ in range(3)]):
            for op, v in (("add", (a + b) % P), ("sub", (a - b) % P), ("mul", a * b % P)):
                lines.append(f"{op} {_h(a)} {_h(b)}")
                want.append(_h(v))
        lines.append(f"sqr {_h(a)}")
        want.append(_h(a * a % P))
        lines.append(f"inv {_h(a)}")
        want.append(_h(pow(a, P - 2, P)))
    assert run(lines) == want


def _all8(sign):
    """The scalar whose recoded digits d_0..d_62 are all `sign` * 8 (and d_63 = 8 for +8, i.e. below 2^255)."""
    if sign > 0:
        return sum(8 * 16**i for i in range(64))
    return 8 * 16**63 - sum(8 * 16**i for i in range(63))


def _scalars():
    rng = random.Random(7)
    ks = [1, 2, 3, 8, 9, 16, N - 1, N - 2, N - 8, N // 2, N // 2 + 1, 2**255 - 1, 2**255, _all8(1), _all8(-1),
          N - _all8(1), N - _all8(-1)]
    return ks + [rng.randrange(1, N) for _ in range(24)]


def test_fixed_and_variable_base(run):
    rng = random.Random(11)
    ks = _scalars()
    lines, want = [], []
    for k in ks:
        kp = mul(k, G)
        lines.append(f"base {_h(k)}")
        want.append("0 " + enc(kp).hex())
        pt = mul(rng.randrange(1, N), G)
        lines.append(f"shared {_h(k)} {enc(pt).hex()}")
        want.append("0 " + _h(mul(k, pt)[0]))
        lines.append(f"shared {_h(k)} {enc(G).hex()}")
        want.append("0 " + _h(kp[0]))
    assert run(lines) == want


def test_scalar_and_point_checks(run):
    ks = {0: 0, 1: 1, N - 1: 1, N: 0, N + 1: 0, 2**256 - 1: 0}
    lines = [f"scalar {_h(k)}" for k in ks]
    assert run(lines) == [str(v) for v in ks.values()]
    g = enc(G)
    x, y = G
    bad = {
        "off curve": b"\x04" + x.to_bytes(32, "big") + ((y + 1) % P).to_bytes(32, "big"),
        "X = p": b"\x04" + P.to_bytes(32, "big") + y.to_bytes(32, "big"),
        "Y = p": b"\x04" + x.to_bytes(32, "big") + P.to_bytes(32, "big"),
        "X = p + x": b"\x04" + (P + x).to_bytes(32, "big") + y.to_bytes(32, "big") if P + x < 2**256 else None,
        "zero": bytes(65),
        "zero coordinates": b"\x04" + bytes(64),
        "all ones": b"\xff" * 65,
    }
    for pre in (0x00, 0x02, 0x03, 0x05):
        bad[f"prefix {pre:#x}"] = bytes([pre]) + g[1:]
    good = [g, enc(mul(N - 1, G)), enc(mul(2, G))]
    lines = [f"point {b.hex()}" for b in bad.values() if b is not None] + [f"point {b.hex()}" for b in good]
    want = ["0"] * sum(b is not None for b in bad.values()) + ["1"] * len(good)
    assert run(lines) == want
    # the operations report them through the status bits and write zeros
    z65, z32 = "00" * 65, "00" * 32
    lines = [f"base {_h(0)}", f"base {_h(N)}", f"base {(b'\xff' * 32).hex()}",
             f"shared {_h(5)} {bad['off curve'].hex()}", f"shared {_h(N)} {g.hex()}",
             f"shared {_h(0)} {bad['prefix 0x2'].hex()}"]
    assert run(lines) == ["2 " + z65, "2 " + z65, "2 " + z65, "1 " + z32, "2 " + z32, "3 " + z32]
