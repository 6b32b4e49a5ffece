"""The threshold RSA code of circl_b200/csrc/rsa.cuh compiled for the host (g++, no GPU) through
tests/cpp/test_tssrsa_host.cpp, against tests/tssrsa_model.py and Python integers: mod_inverse at 64, 96 and 128 words
on invertible and non-invertible values, tss_lambda on every index set of size <= 4 over {0..7} and on random sets of
64 indices up to 65535, the Bezout pair of (4 Delta^2, e), and whole SignShare and Combine on their edge classes."""
import itertools
import os
import random
import subprocess

import pytest

import brsa_model as bm
import tssrsa_model as tm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def run(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("tssrsa") / "tssrsa_host")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Wno-unknown-pragmas",
                        os.path.join(ROOT, "tests", "cpp", "test_tssrsa_host.cpp"), "-o", path],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]

    def go(lines):
        out = subprocess.run([path], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=900)
        assert out.returncode == 0, out.stderr
        res = out.stdout.splitlines()
        assert len(res) == len(lines)
        return res
    return go


def _hx(x, n=None):
    n = n if n is not None else (x.bit_length() + 7) // 8 or 1
    return x.to_bytes(n, "big").hex()


def _wn(k):
    return next(w for w in (64, 96, 128) if k.n.bit_length() <= 32 * w)


@pytest.mark.parametrize("name", ["rsa2048", "rsa3072", "rsa4096"])
def test_mod_inverse(run, name):
    k = bm.all_keys()[name]
    w, n = _wn(k), k.n
    rng = random.Random(name)
    xs = [1, 2, n - 1, n - 2] + [rng.randrange(1, n) for _ in range(20)]
    bad = [0, n, k.p, 2 * k.p, k.q, k.p * rng.randrange(1, k.q)]
    lines = [f"inv {w} {_hx(n)} {_hx(x)}" for x in xs + bad]
    want = [_hx(pow(x, -1, n), 4 * w) for x in xs] + ["none"] * len(bad)
    assert run(lines) == want


def _lambda_want(l, S):
    dlt = tm.delta(l)
    out = []
    for j in S:
        lam = tm.compute_lambda(dlt, S, 0, j, l)
        if lam is None:
            return "1"
        out.append(("-" if lam < 0 else "+") + _hx(abs(lam), 4 * 41))
    return " ".join(["0"] + out)


def test_lambda_small_sets(run):
    lines, want = [], []
    for l in (3, 5, 7):
        for size in range(1, 5):
            for S in itertools.product(range(8), repeat=size):  # repeats included: the reference accepts them
                lines.append(f"lambda {l} {','.join(map(str, S))}")
                want.append(_lambda_want(l, list(S)))
    assert run(lines) == want


def test_lambda_large_sets(run):
    rng = random.Random(64)
    lines, want = [], []
    for _ in range(40):
        S = rng.sample(range(1, 65536), 64)
        lines.append(f"lambda 64 {','.join(map(str, S))}")
        want.append(_lambda_want(64, S))
    for l in (32, 64):  # 1..l: lambda is always an integer, and the largest Delta
        S = list(range(1, l + 1))
        rng.shuffle(S)
        lines.append(f"lambda {l} {','.join(map(str, S))}")
        want.append(_lambda_want(l, S))
    assert run(lines) == want


def test_reference_lambdas(run):
    for c in tm.reference_data()["lambda"]:
        if c["i"] == 0:
            got = run([f"lambda {c['l']} {','.join(map(str, c['S']))}"])[0].split()
            t = c["S"].index(c["j"])
            v = int(got[1 + t][1:], 16) * (-1 if got[1 + t][0] == "-" else 1)
            assert v == int(c["want"])


def test_bezout(run):
    lines, want = [], []
    for l in (2, 3, 5, 16, 64):
        for e in (3, 5, 17, 65537, 0xffffffff, 4294967291):
            ep = 4 * tm.delta(l) ** 2
            _, a, b = tm.go_gcd(ep, e)
            lines.append(f"bezout {l} {e}")
            want.append(f"{'-' if a < 0 else '+'}{_hx(abs(a), 4)} {'-' if b < 0 else '+'}{_hx(abs(b), 4 * 19)}")
    assert run(lines) == want


def _deal(k, players, threshold, rng):
    class S:
        def read(self, n):
            return rng.randbytes(n)
    return tm.deal(S(), players, threshold, k.p, k.q, k.e)


@pytest.mark.parametrize("name", ["rsa2048", "rsa3000u", "rsa4096"])
def test_sign_share(run, name):
    k = bm.all_keys()[name]
    w, kl = _wn(k), k.klen
    rng = random.Random(name)
    players = 5
    si = _deal(k, players, 3, rng)
    ebits = k.n.bit_length() - 2 + (2 * tm.delta(players)).bit_length()
    lines, want = [], []
    xs = [0, 1, k.n - 1, k.n, k.n + 1, (1 << (8 * kl)) - 1, rng.randrange(k.n)]
    for i, s in enumerate(si[:2]):
        E = 2 * tm.delta(players) * s
        for x in xs:
            lines.append(f"sign {w} {_hx(k.n)} {ebits} {_hx(E)} {_hx(x, kl)}")
            want.append(_hx(pow(x, E, k.n), kl))
    E = (1 << ebits) - 1  # the largest cached value the bound admits
    lines.append(f"sign {w} {_hx(k.n)} {ebits} {_hx(E)} {_hx(xs[-1], kl)}")
    want.append(_hx(pow(xs[-1], E, k.n), kl))
    assert run(lines) == want


def _combine_lines(k, players, ops):
    w, kl = _wn(k), k.klen
    lines, want = [], []
    for idx, xi, x in ops:
        lines.append(f"combine {w} {_hx(k.n)} {k.e:x} {players} {','.join(map(str, idx))} "
                     f"{b''.join(v.to_bytes(kl, 'big') for v in xi).hex()} {_hx(x, kl)}")
        st, y = tm.combine(k.n, k.e, players, idx, xi, x)
        want.append(f"{st} {_hx(y, kl)}")
    return lines, want


def edge_ops(k, players, threshold, rng):
    """(idx, xi, x) of every edge class: honest rows, bad index sets, corrupted and degenerate shares, edge x"""
    s = _deal(k, players, threshold, rng)
    E = [2 * tm.delta(players) * v for v in s]
    kl = k.klen

    def honest(idx, x):
        return list(idx), [pow(x, E[j - 1], k.n) for j in idx], x
    x = rng.randrange(k.n)
    ops = [honest(rng.sample(range(1, players + 1), threshold), x),
           honest(range(1, players + 1), rng.randrange(k.n))]
    i0 = honest(range(1, threshold + 1), x)
    ops.append(([0] + i0[0][1:], i0[1], x))  # index 0
    ops.append(([i0[0][0]] * threshold, [i0[1][0]] * threshold, x))  # a repeated index
    if players == 3:
        ops.append(([1, 3 + 2], [i0[1][0], i0[1][-1]], x))  # {1, 5}: lambda not an integer
        ops.append(([2, 4], [i0[1][0], i0[1][-1]], x))  # {2, 4}: integral, wrong
    bad = honest(range(1, threshold + 1), x)
    bad[1][-1] ^= 1 << 40  # corrupted xi
    ops.append(bad)
    for v in (0, k.p, k.q * 3):  # xi = 0 and xi = 0 mod a prime: no inverse
        op = honest(range(1, threshold + 1), x)
        op[1][0] = v
        ops.append(op)
        op = honest(range(1, threshold + 1), x)
        op[1][-1] = v
        ops.append(op)
    for xv in (0, 1, k.n - 1, k.n, k.n + 1, k.p, 2 * k.q, (1 << (8 * kl)) - 1):
        ops.append(honest(range(1, threshold + 1), xv))
    return ops


@pytest.mark.parametrize("name,players,threshold", [("rsa2048", 3, 2), ("rsa2048e3", 3, 2), ("rsa2048", 7, 4),
                                                    ("rsa3072", 3, 2), ("rsa4096", 5, 3)])
def test_combine_edge_classes(run, name, players, threshold):
    k = bm.all_keys()[name]
    rng = random.Random(name + str(players))
    lines, want = _combine_lines(k, players, edge_ops(k, players, threshold, rng))
    got = run(lines)
    assert got == want
    assert {w.split()[0] for w in want} == {"0", "1", "2"}
