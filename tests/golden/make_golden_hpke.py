#!/usr/bin/env python3
"""Extract the KEM fields of CIRCL's RFC 9180 test vectors into tests/golden/hpke_vectors.json.gz (data only; nothing
of CIRCL is executed).  Usage:   python tests/golden/make_golden_hpke.py <path of a CIRCL checkout>

  hpke/testdata/vectors_rfc9180_5f503c5.json.gz   every vector with kem_id 0x20 (DHKEM(X25519, HKDF-SHA256)) or
                                                  0x21 (DHKEM(X448, HKDF-SHA512)), all four modes; per vector the
                                                  mode, kem_id, ikm / sk / pk of E, R and S (S in the auth modes),
                                                  enc and shared_secret
"""
import gzip
import json
import os
import sys

OUT = os.path.dirname(os.path.abspath(__file__))
SRC = "hpke/testdata/vectors_rfc9180_5f503c5.json.gz"
FIELDS = ("mode", "kem_id", "ikmE", "skEm", "pkEm", "ikmR", "skRm", "pkRm", "ikmS", "skSm", "pkSm", "enc", "shared_secret")


def hpke_vectors(circl):
    vs = json.load(gzip.open(os.path.join(circl, SRC)))
    keep = [{f: v[f] for f in FIELDS if f in v} for v in vs if v["kem_id"] in (0x20, 0x21)]
    out = {"source": SRC, "vectors": keep}
    raw = json.dumps(out, separators=(",", ":"), sort_keys=True).encode()
    path = os.path.join(OUT, "hpke_vectors.json.gz")
    with gzip.GzipFile(path, "wb", mtime=0) as f:
        f.write(raw)
    print(f"hpke_vectors.json.gz: {len(keep)} vectors, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    hpke_vectors(sys.argv[1])
