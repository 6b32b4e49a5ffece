#!/usr/bin/env python3
"""Extract the reference's Ed448 test data into tests/golden/ed448_vectors.json.gz (data only; nothing of the reference
is executed).  Run in the build container, which has the reference:   python tests/golden/make_golden_ed448.py

  sign/ed448/rfc8032_test.go                      the pure-Ed448 vectors of RFC 8032 section 7.4 (vectorsEd448 entries
                                                  with scheme "Ed448Pure", one of them with a context); the two
                                                  Ed448ph vectors are left out
  sign/ed448/testdata/wycheproof_Ed448.json.gz    the Wycheproof tests; valid = (result == "valid"), as
                                                  wycheproof_test.go reads them
"""
import gzip
import json
import os
import re

REF = "/root/reference"
OUT = os.path.dirname(os.path.abspath(__file__))


def _bytes(block, field):
    m = re.search(r"\b" + field + r":\s*\[\]byte\{(.*?)\}", block, re.S)
    return bytes(int(x, 16) for x in re.findall(r"0x([0-9a-fA-F]{2})", m.group(1))).hex()


def rfc8032():
    src = open(os.path.join(REF, "sign/ed448/rfc8032_test.go")).read()
    body = src[src.index("var vectorsEd448"):]
    out = []
    for block in re.split(r"\n\t\{\n", body)[1:]:
        if re.search(r'scheme:\s*"([^"]*)"', block).group(1) != "Ed448Pure":
            continue
        out.append({"name": re.search(r'name:\s*"([^"]*)"', block).group(1).strip("-"), "seed": _bytes(block, "sk"),
                    "pk": _bytes(block, "pk"), "msg": _bytes(block, "msg"), "sig": _bytes(block, "sig"),
                    "ctx": _bytes(block, "ctx")})
    return out


def wycheproof():
    w = json.load(gzip.open(os.path.join(REF, "sign/ed448/testdata/wycheproof_Ed448.json.gz")))
    out = []
    for g in w["testGroups"]:
        for t in g["tests"]:
            out.append({"tcId": t["tcId"], "seed": g["key"]["sk"], "pk": g["key"]["pk"], "msg": t["msg"], "sig": t["sig"],
                        "valid": t["result"] == "valid"})
    return out


def main():
    out = {"source": "sign/ed448/rfc8032_test.go, sign/ed448/testdata/wycheproof_Ed448.json.gz",
           "rfc8032": rfc8032(), "wycheproof": wycheproof()}
    raw = json.dumps(out, separators=(",", ":"), sort_keys=True).encode()
    path = os.path.join(OUT, "ed448_vectors.json.gz")
    with gzip.GzipFile(path, "wb", mtime=0) as f:
        f.write(raw)
    print(f"ed448_vectors.json.gz: {os.path.getsize(path)} bytes, {len(out['rfc8032'])} RFC 8032, "
          f"{len(out['wycheproof'])} Wycheproof")


if __name__ == "__main__":
    main()
