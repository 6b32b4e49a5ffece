"""Threshold RSA rates (tss/rsa) on one GPU, device-resident, at 2048, 3072 and 4096 bits under the fixture keys of
tests/golden/brsa_keys.json.gz: SignShare (x^(2 Delta s_i) mod N) of random digests below N at players = 3, and Combine
of honest shares at (players, k) = (3, 2) and (16, 9), every op combining the shares of indices 1 .. k.  Beside them,
in the same run, blind RSA BlindSign (cb200_brsa_blind_sign) under the same key at the same batch size.  SignShare and
BlindSign batches are 2^15 ops, Combine batches 2^14.  CUDA events around `steps` calls after `warmup` calls, repeated
`repeats` times: each rate is the median of the repeats, with their minimum and maximum beside it (`*_spread`).  Prints
one JSON object with the card name and its power limit, read in the same run.

  python scripts/bench_tssrsa.py [--steps 2] [--warmup 1] [--repeats 3]
"""
import argparse
import json
import math
import os
import random
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

SIZES = [(2048, "rsa2048"), (3072, "rsa3072"), (4096, "rsa4096")]
SIGN_BATCH, COMBINE_BATCH = 1 << 15, 1 << 14


def timed(fn, steps, warm):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def put(line, name, rates):
    rs = sorted(rates)
    line[name + "_per_s"] = round(rs[len(rs) // 2])
    line[name + "_spread"] = [round(rs[0]), round(rs[-1])]


def _be(x):
    return x.to_bytes((x.bit_length() + 7) // 8, "big")


class _Stream:
    def __init__(self, rng):
        self.rng = rng

    def read(self, n):
        return self.rng.randbytes(n)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    import brsa_model as bm
    import tssrsa_model as tm
    import circl_b200
    from circl_b200._ffi import check, lib
    circl_b200.init(0)
    L = lib()
    check(L.cb200_set_stream(torch.cuda.current_stream().cuda_stream))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=30).stdout.strip().splitlines()
    res = {"card": q[0] if q else "unknown", "sign_batch": SIGN_BATCH, "combine_batch": COMBINE_BATCH,
           "steps": a.steps, "warmup": a.warmup, "repeats": a.repeats}
    keys = bm.all_keys()
    rng = np.random.default_rng(1)
    st = torch.empty((SIGN_BATCH,), dtype=torch.uint8, device="cuda")
    for bits, name in SIZES:
        k = keys[name]
        assert k.n.bit_length() == bits
        kl, n = k.klen, SIGN_BATCH
        line = {}
        c = torch.from_numpy(rng.integers(0, 256, size=(n, kl), dtype=np.uint8)).cuda()
        c[:, 0] = 0  # below N
        out = torch.empty_like(c)
        nb, eb = _be(k.n), _be(k.e)

        def shares(players, threshold):
            return tm.deal(_Stream(random.Random(bits + players)), players, threshold, k.p, k.q, k.e)

        s3 = shares(3, 2)
        E = _be(2 * math.factorial(3) * s3[0])

        def sign():
            check(L.cb200_tssrsa_sign_share(nb, len(nb), 3, E, len(E), c.data_ptr(), out.data_ptr(), n))
        put(line, "sign_share", [n / timed(sign, a.steps, a.warmup) * 1e3 for _ in range(a.repeats)])
        assert int.from_bytes(out[5].cpu().numpy().tobytes(), "big") == pow(
            int.from_bytes(c[5].cpu().numpy().tobytes(), "big"), 2 * 6 * s3[0], k.n)
        dp, dq, qinv = k.crt()
        bargs = [x for f in (nb, eb, _be(k.p), _be(k.q), _be(dp), _be(dq), _be(qinv)) for x in (f, len(f))]

        def b_sign():
            check(L.cb200_brsa_blind_sign(*bargs, c.data_ptr(), out.data_ptr(), st.data_ptr(), n))
        put(line, "brsa_blind_sign", [n / timed(b_sign, a.steps, a.warmup) * 1e3 for _ in range(a.repeats)])
        assert not st.any().item()
        line["blind_sign_over_sign_share"] = round(line["brsa_blind_sign_per_s"] / line["sign_share_per_s"], 2)
        m = COMBINE_BATCH
        x = c[:m]
        for players, kk in ((3, 2), (16, 9)):
            s = shares(players, kk)
            xi = torch.empty((m, kk, kl), dtype=torch.uint8, device="cuda")
            for j in range(kk):
                Ej = _be(2 * math.factorial(players) * s[j])
                check(L.cb200_tssrsa_sign_share(nb, len(nb), players, Ej, len(Ej), x.data_ptr(), out.data_ptr(), m))
                xi[:, j].copy_(out[:m])
            idx = torch.arange(1, kk + 1, dtype=torch.int16, device="cuda").repeat(m, 1).contiguous()
            sig = torch.empty((m, kl), dtype=torch.uint8, device="cuda")

            def comb():
                check(L.cb200_tssrsa_combine(nb, len(nb), eb, len(eb), players, kk, kk, idx.data_ptr(),
                                             xi.data_ptr(), x.data_ptr(), sig.data_ptr(), st.data_ptr(), m))
            put(line, f"combine_{players}_{kk}", [m / timed(comb, a.steps, a.warmup) * 1e3 for _ in range(a.repeats)])
            assert not st[:m].any().item()
            y = int.from_bytes(sig[7].cpu().numpy().tobytes(), "big")
            assert pow(y, k.e, k.n) == int.from_bytes(x[7].cpu().numpy().tobytes(), "big")
        res[f"rsa{bits}"] = line
    circl_b200.shutdown()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
