#!/usr/bin/env python3
"""Write tests/golden/tssrsa_reference.json.gz: the data of the reference's tss/rsa tests, as data (nothing of CIRCL is
executed or copied).  Usage:   python tests/golden/make_golden_tssrsa.py

  deal            TestDeal: p = 23, q = 11, e = 3, players 3, threshold 2, the byte stream {33, 17} -> s = 15, 48, 26
  sign            TestKeyShare_Sign: N = 253, players 3, s = 15, x = 150 -> xi = 243
  lambda          TestComputeLambda (S = 1..5, l = 5, j = 3 -> 1200) and TestComputeLambdaLarge (S = {7, 14, 21},
                  l = 32, j = 7, four values of i)
  check_indices   TestCheckIndices: S = {1, 4}, l = 8, the (i, j) pairs and the expected answer
  delta           TestCalculateDelta: 0 -> 1, 1 -> 1, 5 -> 120
  untrusted       TestCombineSignSharesRejectsUntrustedParameters: the SignShare encoding, N = 3233, e = 17,
                  players 3, threshold 1, msg {1}, and the expected error
  keyshare_ok / signshare_ok        TestMarshallKeyShare / TestMarshallSignShare round trips (fields, hex)
  keyshare_bad / signshare_bad      encodings UnmarshalBinary must refuse (hex)
  keyshare_wrap / signshare_wrap    TestUnmarshal*BoundsWrap: siLen / xiLen of 65528, 65534 and 65535 in an 8 + len
                                    byte buffer with byte 8 set: KeyShare refuses all three, SignShare accepts all three
"""
import gzip
import json
import os

OUT = os.path.dirname(os.path.abspath(__file__))


def main():
    data = {
        "deal": {"p": 23, "q": 11, "e": 3, "players": 3, "threshold": 2, "stream": [33, 17], "si": [15, 48, 26]},
        "sign": {"n": 253, "players": 3, "si": 15, "index": 1, "x": 150, "xi": 243},
        "lambda": [
            {"S": [1, 2, 3, 4, 5], "l": 5, "i": 0, "j": 3, "want": "1200"},
            {"S": [7, 14, 21], "l": 32, "i": 0, "j": 7, "want": "789392510801080590501654036480000000"},
            {"S": [7, 14, 21], "l": 32, "i": 12, "j": 7, "want": "48330153722515138193978818560000000"},
            {"S": [7, 14, 21], "l": 32, "i": 19, "j": 7, "want": "-26850085401397298996654899200000000"},
            {"S": [7, 14, 21], "l": 32, "i": 32, "j": 7, "want": "531631690947666520133767004160000000"},
        ],
        "check_indices": {
            "S": [1, 4], "l": 8,
            "true": [[0, 1], [0, 4], [2, 1], [2, 4], [3, 1], [3, 4], [5, 1], [5, 4], [6, 1], [6, 4], [8, 1], [8, 4]],
            "false": [[1, 1], [1, 4], [4, 1], [4, 4], [9, 1], [9, 4], [-1, 1], [-1, 4], [0, 0], [0, 2], [0, 3]],
        },
        "delta": [[0, 1], [1, 1], [5, 120]],
        "untrusted": {"share": "ffff00010001000102", "n": 3233, "e": 17, "players": 3, "threshold": 1,
                      "msg": "01", "error": "rsa_threshold: share players did not match protocol players"},
        "keyshare_ok": [
            {"si": 10, "twoDeltaSi": 20, "index": 30, "threshold": 10, "players": 2},
            {"si": 10, "twoDeltaSi": None, "index": 30, "threshold": 0, "players": 200},
            {"si": 0, "twoDeltaSi": 0, "index": 0, "threshold": 0, "players": 0},
        ],
        "keyshare_bad": ["", "010001", "000100010001", "0001000100010001", "00010001000100", "000100010001000201",
                         "0001000100010001010100", "000100010001000101010001"],
        "signshare_ok": [
            {"xi": 10, "index": 30, "players": 16, "threshold": 18},
            {"xi": 0, "index": 0, "players": 0, "threshold": 0},
        ],
        "signshare_bad": ["", "000000", "0000000000000000", "0000000000000001", "000000000000000201"],
        "keyshare_wrap": [65528, 65534, 65535],
        "signshare_wrap": [65528, 65534, 65535],
    }
    with gzip.GzipFile(os.path.join(OUT, "tssrsa_reference.json.gz"), "wb", mtime=0) as f:
        f.write(json.dumps(data, sort_keys=True).encode())


if __name__ == "__main__":
    main()
