#!/usr/bin/env python3
"""Extract the reference's Ed25519 test data into tests/golden/ed25519_vectors.json.gz (data only; nothing of the
reference is executed).  Run in the build container, which has the reference:   python tests/golden/make_golden_ed25519.py

  sign/ed25519/rfc8032_test.go                      the pure-Ed25519 vectors of RFC 8032 section 7.1 (vectorsEd25519
                                                    entries with scheme "Ed25519Pure")
  sign/ed25519/testdata/sign.input.txt.gz           the 1024 lines of TestRFC8032 (seed||pk : pk : msg : sig||msg)
  sign/ed25519/testdata/wycheproof_Ed25519.json.gz  the Wycheproof tests; valid = (result == "valid"), as
                                                    wycheproof_test.go:68 reads them
"""
import gzip
import json
import os
import re

REF = "/root/reference"
OUT = os.path.dirname(os.path.abspath(__file__))


def _bytes(block, field):
    m = re.search(field + r":\s*\[\]byte\{(.*?)\}", block, re.S)
    return bytes(int(x, 16) for x in re.findall(r"0x([0-9a-fA-F]{2})", m.group(1))).hex()


def rfc8032():
    src = open(os.path.join(REF, "sign/ed25519/rfc8032_test.go")).read()
    body = src[src.index("var vectorsEd25519"):]
    out = []
    for block in re.split(r"\n\t\{\n", body)[1:]:
        if re.search(r'scheme:\s*"([^"]*)"', block).group(1) != "Ed25519Pure":
            continue
        out.append({"name": re.search(r'name:\s*"([^"]*)"', block).group(1).strip("-"), "seed": _bytes(block, "sk"),
                    "pk": _bytes(block, "pk"), "msg": _bytes(block, "msg"), "sig": _bytes(block, "sig")})
    return out


def sign_input():
    out = []
    for line in gzip.open(os.path.join(REF, "sign/ed25519/testdata/sign.input.txt.gz")).read().decode().splitlines():
        v = line.split(":")
        out.append({"seed": v[0][:64], "pk": v[1], "msg": v[2], "sig": v[3][:128]})
    return out


def wycheproof():
    w = json.load(gzip.open(os.path.join(REF, "sign/ed25519/testdata/wycheproof_Ed25519.json.gz")))
    out = []
    for g in w["testGroups"]:
        for t in g["tests"]:
            out.append({"tcId": t["tcId"], "seed": g["key"]["sk"], "pk": g["key"]["pk"], "msg": t["msg"], "sig": t["sig"],
                        "valid": t["result"] == "valid"})
    return out


def main():
    out = {"source": "sign/ed25519/rfc8032_test.go, sign/ed25519/testdata/{sign.input.txt,wycheproof_Ed25519.json}.gz",
           "rfc8032": rfc8032(), "sign_input": sign_input(), "wycheproof": wycheproof()}
    raw = json.dumps(out, separators=(",", ":"), sort_keys=True).encode()
    path = os.path.join(OUT, "ed25519_vectors.json.gz")
    with gzip.GzipFile(path, "wb", mtime=0) as f:
        f.write(raw)
    print(f"ed25519_vectors.json.gz: {os.path.getsize(path)} bytes, {len(out['rfc8032'])} RFC 8032, "
          f"{len(out['sign_input'])} sign.input, {len(out['wycheproof'])} Wycheproof")


if __name__ == "__main__":
    main()
