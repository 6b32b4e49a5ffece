#!/usr/bin/env python3
"""Write the partially blind RSA fixture tests/golden/pbrsa_keys.json.gz (data only; nothing of CIRCL is executed).
Usage:   python tests/golden/make_golden_pbrsa.py <path of a CIRCL checkout>

Every key is two safe primes (p = 2 p' + 1 with p' prime, so p = 3 mod 4), e = 65537, as n, e, d, p, q in hex:
  strong2048   the strong key of blindsign/blindrsa/partiallyblindrsa/pbrsa_test.go (loadStrongRSAKey), its hex
               values copied as they are: two 1024-bit primes
  safe3072     two 1536-bit primes
  safe4096     two 2048-bit primes (e' then has 2046 bits)
  safe2050     a 2050-bit modulus: lambda = 1025, lambda mod 8 = 1, so the clear of bit lambda - 2 is inside e'
  safe2052     a 2052-bit modulus: lambda = 1026, lambda mod 8 = 2, both clears fall above e'
  safe3073     a 3073-bit modulus: emBits = 3072 = 0 mod 8, the top byte of s^e' mod N must be zero
  safe2048u    primes of 1088 and 960 bits: e' (1022 bits) exceeds q' and is reduced mod q'
The safe primes come from `openssl prime -generate -safe`, which sets the top two bits, so the bit length of each
modulus is the sum of its primes' bit lengths.  The tests never run this script.
"""
import concurrent.futures as cf
import gzip
import json
import os
import re
import subprocess
import sys

OUT = os.path.dirname(os.path.abspath(__file__))
SPECS = {"safe3072": (1536, 1536), "safe4096": (2048, 2048), "safe2050": (1025, 1025), "safe2052": (1026, 1026),
         "safe3073": (1537, 1536), "safe2048u": (1088, 960)}
E = 65537


def safe_prime(bits):
    out = subprocess.run(["openssl", "prime", "-generate", "-safe", "-hex", "-bits", str(bits)], check=True,
                         capture_output=True, text=True).stdout
    return int(out.strip(), 16)


def entry(n, p, q, d=None):
    assert p * q == n and p % 4 == 3 and q % 4 == 3
    d = d if d is not None else pow(E, -1, (p - 1) * (q - 1))
    return {k: hex(v) for k, v in (("n", n), ("e", E), ("d", d), ("p", p), ("q", q))}


def strong_key(circl):
    src = open(os.path.join(circl, "blindsign", "blindrsa", "partiallyblindrsa", "pbrsa_test.go")).read()
    body = src[src.index("func loadStrongRSAKey"):]
    v = {k: int(re.search(k + r'Enc := "([0-9a-f]+)"', body).group(1), 16) for k in ("p", "q", "N", "e", "d")}
    assert v["e"] == E
    return entry(v["N"], v["p"], v["q"], v["d"])


def main(circl):
    keys = {"strong2048": strong_key(circl)}
    with cf.ThreadPoolExecutor(max_workers=os.cpu_count()) as ex:
        futs = {name: (ex.submit(safe_prime, a), ex.submit(safe_prime, b)) for name, (a, b) in SPECS.items()}
        for name, (a, b) in SPECS.items():
            p, q = futs[name][0].result(), futs[name][1].result()
            assert p != q and (p * q).bit_length() == a + b, name
            keys[name] = entry(p * q, p, q)
    raw = json.dumps(keys, separators=(",", ":"), sort_keys=True).encode()
    with gzip.GzipFile(os.path.join(OUT, "pbrsa_keys.json.gz"), "wb", mtime=0) as f:
        f.write(raw)
    print("pbrsa_keys.json.gz:", ", ".join(f"{k} {int(v['n'], 16).bit_length()} bits" for k, v in keys.items()))


if __name__ == "__main__":
    main(sys.argv[1])
