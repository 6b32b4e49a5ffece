#!/usr/bin/env python3
"""Write tests/golden/hpke_p521_vectors.json.gz for DHKEM(P-521, HKDF-SHA512) (data only; nothing of CIRCL is executed).
Usage:   python tests/golden/make_golden_hpke_p521.py <path of a CIRCL checkout>

  vectors     the KEM fields of every vector of hpke/testdata/vectors_rfc9180_5f503c5.json.gz with kem_id 0x12, all
              four modes (mode, kem_id, ikm / sk / pk of E, R and S, enc, shared_secret)
The file has no vector for kem_id 0x11 (P-384), which the tests pin against a live model instead.
"""
import gzip
import json
import os
import sys

OUT = os.path.dirname(os.path.abspath(__file__))
SRC = "hpke/testdata/vectors_rfc9180_5f503c5.json.gz"
FIELDS = ("mode", "kem_id", "ikmE", "skEm", "pkEm", "ikmR", "skRm", "pkRm", "ikmS", "skSm", "pkSm", "enc", "shared_secret")


def main(circl):
    vs = json.load(gzip.open(os.path.join(circl, SRC)))
    keep = [{f: v[f] for f in FIELDS if f in v} for v in vs if v["kem_id"] == 0x12]
    assert not any(v["kem_id"] == 0x11 for v in vs)
    out = {"source": SRC, "vectors": keep}
    raw = json.dumps(out, separators=(",", ":"), sort_keys=True).encode()
    path = os.path.join(OUT, "hpke_p521_vectors.json.gz")
    with gzip.GzipFile(path, "wb", mtime=0) as f:
        f.write(raw)
    print(f"hpke_p521_vectors.json.gz: {len(keep)} vectors, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main(sys.argv[1])
