#!/usr/bin/env python3
"""Write tests/golden/hpke_p256_vectors.json.gz for DHKEM(P-256, HKDF-SHA256) (data only; nothing of CIRCL is executed).
Usage:   python tests/golden/make_golden_hpke_p256.py <path of a CIRCL checkout> [--ctr-seed HEX ...]

  vectors     the KEM fields of every vector of hpke/testdata/vectors_rfc9180_5f503c5.json.gz with kem_id 0x10, all
              four modes (mode, kem_id, ikm / sk / pk of E, R and S, enc, shared_secret)
  ctr_seeds   DeriveKeyPair seeds whose first candidate (ctr = 0) is not below n, so that the key comes from a later
              candidate, with the oracle's key pair and counter.  About one seed in 2^32 qualifies; they are found by
              p256_ctr_search.c (OpenSSL's SHA-256 on every core; a few minutes) unless given with --ctr-seed.
"""
import gzip
import json
import os
import subprocess
import sys
import tempfile

OUT = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(OUT))
SRC = "hpke/testdata/vectors_rfc9180_5f503c5.json.gz"
FIELDS = ("mode", "kem_id", "ikmE", "skEm", "pkEm", "ikmR", "skRm", "pkRm", "ikmS", "skSm", "pkSm", "enc", "shared_secret")
PREFIX = b"hpke p256 candidate loop"  # the first 24 bytes of every searched seed


def search(count):
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "search")
        subprocess.run(["cc", "-O2", "-pthread", "-Wno-deprecated-declarations", os.path.join(OUT, "p256_ctr_search.c"),
                        "-o", exe, "-lcrypto"], check=True)
        out = subprocess.run([exe, PREFIX.hex(), str(os.cpu_count()), str(count)], check=True, capture_output=True,
                             text=True).stdout
    return sorted(out.split())


def main(circl, seeds):
    sys.path.insert(0, ROOT)
    from oracle import p256 as oracle_p256
    vs = json.load(gzip.open(os.path.join(circl, SRC)))
    keep = [{f: v[f] for f in FIELDS if f in v} for v in vs if v["kem_id"] == 0x10]
    ctr = []
    for s in seeds or search(1):
        pk, sk, c = oracle_p256.keygen(bytes.fromhex(s))
        assert c > 0, s
        ctr.append({"ikm": s, "ctr": c, "sk": sk.hex(), "pk": pk.hex()})
    out = {"source": SRC, "vectors": keep, "ctr_seeds": ctr}
    raw = json.dumps(out, separators=(",", ":"), sort_keys=True).encode()
    path = os.path.join(OUT, "hpke_p256_vectors.json.gz")
    with gzip.GzipFile(path, "wb", mtime=0) as f:
        f.write(raw)
    print(f"hpke_p256_vectors.json.gz: {len(keep)} vectors, {len(ctr)} ctr seeds, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    args = sys.argv[1:]
    given = [args[i + 1] for i, a in enumerate(args) if a == "--ctr-seed"]
    main(args[0], given)
