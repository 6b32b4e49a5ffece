#!/usr/bin/env python3
"""Extract the PQCgenKAT transcript hash of FrodoKEM-640-SHAKE into tests/golden/frodo_vectors.json.gz (data only;
nothing of CIRCL is executed).  Usage:   python tests/golden/make_golden_frodo.py <path of a CIRCL checkout>

  kem/frodo/kat_test.go   the scheme name and the SHA-256 of its 100-round transcript (DeriveKeyPair,
                          EncapsulateDeterministically and Decapsulate driven by the NIST DRBG)
"""
import gzip
import json
import os
import re
import sys

OUT = os.path.dirname(os.path.abspath(__file__))
SRC = "kem/frodo/kat_test.go"


def frodo_vectors(circl):
    text = open(os.path.join(circl, SRC)).read()
    kats = [{"name": n, "sha256": h} for n, h in re.findall(r'\{"(FrodoKEM-[^"]+)",\s*"([0-9a-f]{64})"\}', text)]
    assert kats, "no KAT entries found"
    out = {"source": SRC, "rounds": 100, "seed_size": 48, "encapsulation_seed_size": 16, "kats": kats}
    raw = json.dumps(out, separators=(",", ":"), sort_keys=True).encode()
    path = os.path.join(OUT, "frodo_vectors.json.gz")
    with gzip.GzipFile(path, "wb", mtime=0) as f:
        f.write(raw)
    print(f"frodo_vectors.json.gz: {len(kats)} transcript(s), {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    frodo_vectors(sys.argv[1])
