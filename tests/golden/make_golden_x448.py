#!/usr/bin/env python3
"""Extract the reference's X448 test data into tests/golden/x448_vectors.json.gz (data only; nothing of the
reference is executed).  Run in the build container, which has the reference:   python tests/golden/make_golden_x448.py

  dh/x448/testdata/rfc7748_kat_test.json.gz     RFC 7748 section 5.2, the six KAT vectors (key_test.go:23-45)
  dh/x448/testdata/rfc7748_times_test.json.gz   the iterated vectors, 1 and 1000 times; 10^6 is left out, as
                                                key_test.go:69 skips it without -long
"""
import gzip
import json
import os

REF = "/root/reference"
OUT = os.path.dirname(os.path.abspath(__file__))


def x448_vectors():
    td = os.path.join(REF, "dh/x448/testdata")
    out = {"source": "dh/x448/testdata/{rfc7748_kat_test,rfc7748_times_test}.json.gz"}
    out["rfc7748_kat"] = json.load(gzip.open(os.path.join(td, "rfc7748_kat_test.json.gz")))
    out["rfc7748_times"] = [v for v in json.load(gzip.open(os.path.join(td, "rfc7748_times_test.json.gz"))) if v["times"] <= 1000]
    raw = json.dumps(out, separators=(",", ":"), sort_keys=True).encode()
    path = os.path.join(OUT, "x448_vectors.json.gz")
    with gzip.GzipFile(path, "wb", mtime=0) as f:
        f.write(raw)
    print(f"x448_vectors.json.gz: {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    x448_vectors()
