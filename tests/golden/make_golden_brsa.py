#!/usr/bin/env python3
"""Write the RSA blind-signature fixtures under tests/golden/ (data only; nothing of CIRCL is executed).
Usage:   python tests/golden/make_golden_brsa.py <path of a CIRCL checkout>

  brsa_rfc9474.json.gz       blindsign/blindrsa/testdata/test_vectors_rfc9474.json.gz as it is: the four RFC 9474
                             variants under one 4096-bit key
  brsa_rfc9500_2048.pem      blindsign/blindrsa/testdata/testRSA2048.rfc9500.pem as it is: the 2048-bit test key of
                             RFC 9500
  brsa_keys.json.gz          keys derived here from a fixed seed with a Miller-Rabin test (n, e, d, p, q in hex):
                               rsa3072    two 1536-bit primes, e = 65537
                               rsa3073    a 3073-bit modulus (bit length 1 mod 8: the encoded message is kLen - 1
                                          bytes), primes of 1537 and 1536 bits, e = 65537
                               rsa2048e3  e = 3 and unbalanced primes of 1040 and 1008 bits (the CRT halves then use
                                          48 words under a 64-word modulus)
                               rsa2048u   primes of 1600 and 448 bits: 64-word CRT halves under a 64-word modulus
                               rsa3000u   primes of 1600 and 1400 bits: 64-word CRT halves under a 96-word modulus
"""
import gzip
import json
import math
import os
import random
import shutil
import sys

OUT = os.path.dirname(os.path.abspath(__file__))
SMALL = [p for p in range(3, 2000) if all(p % d for d in range(2, int(p ** 0.5) + 1))]


def is_probable_prime(n, rng):
    if n < 2 or any(n % p == 0 for p in SMALL if p < n):
        return n in SMALL
    d, s = n - 1, 0
    while d % 2 == 0:
        d, s = d // 2, s + 1
    for _ in range(40):
        x = pow(rng.randrange(2, n - 1), d, n)
        if x in (1, n - 1):
            continue
        for _ in range(s - 1):
            x = x * x % n
            if x == n - 1:
                break
        else:
            return False
    return True


def prime(bits, e, rng):
    while True:
        p = rng.getrandbits(bits) | (3 << (bits - 2)) | 1
        if (p - 1) % e and is_probable_prime(p, rng):
            return p


def key(pbits, qbits, e, nbits, rng):
    while True:
        p, q = prime(pbits, e, rng), prime(qbits, e, rng)
        n = p * q
        if n.bit_length() == nbits and p != q:
            d = pow(e, -1, (p - 1) * (q - 1) // math.gcd(p - 1, q - 1))
            return {k: hex(v) for k, v in (("n", n), ("e", e), ("d", d), ("p", p), ("q", q))}


def main(circl):
    src = os.path.join(circl, "blindsign", "blindrsa", "testdata")
    shutil.copyfile(os.path.join(src, "test_vectors_rfc9474.json.gz"), os.path.join(OUT, "brsa_rfc9474.json.gz"))
    shutil.copyfile(os.path.join(src, "testRSA2048.rfc9500.pem"), os.path.join(OUT, "brsa_rfc9500_2048.pem"))
    rng = random.Random(9474)
    keys = {"rsa3072": key(1536, 1536, 65537, 3072, rng), "rsa3073": key(1537, 1536, 65537, 3073, rng),
            "rsa2048e3": key(1040, 1008, 3, 2048, rng), "rsa2048u": key(1600, 448, 65537, 2048, rng),
            "rsa3000u": key(1600, 1400, 65537, 3000, rng)}
    raw = json.dumps(keys, separators=(",", ":"), sort_keys=True).encode()
    with gzip.GzipFile(os.path.join(OUT, "brsa_keys.json.gz"), "wb", mtime=0) as f:
        f.write(raw)
    print("brsa_keys.json.gz:", ", ".join(f"{k} {int(v['n'], 16).bit_length()} bits" for k, v in keys.items()))


if __name__ == "__main__":
    main(sys.argv[1])
