"""A pure Python restatement of the reference's tss/rsa package (rsa_threshold.go, keyshare.go, util.go) for the
tests, with Go's math/big semantics where they decide a result:
  ModInverse(g, n)   None when gcd(g, n) != 1 (the receiver is then left unchanged)
  Exp(x, y, m)       for y < 0 inverts x first; with no inverse the receiver keeps its value (0 for a fresh Int)
  GCD(a, b)          the classical extended Euclid coefficients
and the shared fixtures: brsa_keys.json.gz (via brsa_model) and tssrsa_reference.json.gz (the reference tests' data)."""
import gzip
import json
import math
import os

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

ERR_INVALID_CALC, ERR_INTERNAL = 1, 2


def reference_data():
    with gzip.open(os.path.join(GOLDEN, "tssrsa_reference.json.gz")) as f:
        return json.load(f)


def delta(players):
    return math.factorial(max(players, 0))


def go_mod_inverse(g, n):
    g %= n
    if math.gcd(g, n) != 1:
        return None
    return pow(g, -1, n)


def go_exp(x, y, m):
    """z.Exp(x, y, m) for a fresh z (0) and m > 1"""
    if y < 0:
        inv = go_mod_inverse(x, m)
        if inv is None:
            return 0
        return pow(inv, -y, m)
    return pow(x, y, m)


def go_gcd(a, b):
    """(d, x, y) with a x + b y = d: the classical extended Euclid on (a, b)"""
    r0, r1, s0, s1, t0, t1 = a, b, 1, 0, 0, 1
    while r1:
        q = r0 // r1
        r0, r1, s0, s1, t0, t1 = r1, r0 - q * r1, s1, s0 - q * s1, t1, t0 - q * t1
    return r0, s0, t0


def check_indices(i, j, l, S):
    return j in S and 0 <= i <= l and i not in S


def compute_lambda(dlt, S, i, j, l):
    """computeLambda (rsa_threshold.go:315-349): the integer lambda, or None for ErrInvalidCalc"""
    if not check_indices(i, j, l, S):
        return None
    num = den = 1
    for jp in S:
        if jp != j:
            num *= i - jp
            den *= j - jp
    if den == 0:
        return None
    q, r = divmod(abs(dlt * num), abs(den))  # Go's QuoRem truncates toward zero
    if r:
        return None
    return q if (dlt * num < 0) == (den < 0) else -q


def sign_share(N, E, x):
    """KeyShare.Sign: x^E mod N (the blinding does not change it)"""
    return pow(x, E, N)


def combine(N, e, players, idx, xi, x):
    """CombineSignShares after its parameter checks: (status, y) with status 0, ERR_INVALID_CALC or ERR_INTERNAL
    (y = 0 then)"""
    dlt = delta(players)
    w = 1
    for j, s in zip(idx, xi):
        lam = compute_lambda(dlt, list(idx), 0, j, players)
        if lam is None:
            return ERR_INVALID_CALC, 0
        tmp = pow(s, abs(2 * lam), N)
        if lam < 0:
            inv = go_mod_inverse(tmp, N)
            if inv is not None:
                tmp = inv
        w = w * tmp % N
    ep = 4 * dlt * dlt
    _, a, b = go_gcd(ep, e)
    y = go_exp(w, a, N) * go_exp(x, b, N) % N
    if pow(y, e, N) != x:
        return ERR_INTERNAL, 0
    return 0, y


def go_rand_int(stream, m):
    """crypto/rand.Int(stream, m) with stream.read(n) -> bytes"""
    bl = (m - 1).bit_length()
    if bl == 0:
        return 0
    k, b = (bl + 7) // 8, bl % 8 or 8
    while True:
        buf = bytearray(stream.read(k))
        assert len(buf) == k
        buf[0] &= (1 << b) - 1
        v = int.from_bytes(buf, "big")
        if v < m:
            return v


def deal(stream, players, threshold, p, q, e):
    """Deal: the shares s_1 .. s_players"""
    m = ((p - 1) * (q - 1)) >> 2
    d = pow(e, -1, m)
    a = [d] + [go_rand_int(stream, m) for _ in range(threshold - 1)]
    return [sum(c * pow(i, k, m) for k, c in enumerate(a)) % m for i in range(1, players + 1)]
