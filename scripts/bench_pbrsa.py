"""Partially blind RSA rates (RSAPBSSA-SHA384) on one GPU, device-resident, at 2048, 3072 and 4096 bits under one
safe-prime key each (tests/golden/pbrsa_keys.json.gz): BlindSign of random blinded messages and Verify of 64-byte
messages, the ops cycling through 16 distinct 16-byte metadata strings, so every op derives its own key.  Beside each,
in the same run, plain blind RSA (cb200_brsa_*, PSS with a 48-byte salt, e = 65537) under a key of the same size
(tests/golden/brsa_*) at the same batch size.  Every batch is 2^15 ops, about one wave of a 132-SM H100 at these
kernels' 256 resident threads per SM.  CUDA events around `steps` calls after `warmup` calls, repeated `repeats`
times: each rate is the median of the repeats, with their minimum and maximum beside it (`*_spread`).  Prints one JSON
object with the card name and its power limit, read in the same run.

  python scripts/bench_pbrsa.py [--steps 2] [--warmup 1] [--repeats 3]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

# (bits, pbrsa fixture key, brsa fixture key)
SIZES = [(2048, "strong2048", "rsa2048"), (3072, "safe3072", "rsa3072"), (4096, "safe4096", "rsa4096")]
BATCH = 1 << 15


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    import brsa_model as bm
    import pbrsa_model as pm
    import circl_b200
    from circl_b200._ffi import check, lib
    circl_b200.init(0)
    L = lib()
    check(L.cb200_set_stream(torch.cuda.current_stream().cuda_stream))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=30).stdout.strip().splitlines()
    res = {"card": q[0] if q else "unknown", "batch": BATCH, "steps": a.steps, "warmup": a.warmup,
           "repeats": a.repeats, "message_bytes": 64, "metadata": "16 distinct strings of 16 bytes"}
    pkeys, bkeys = pm.keys(), bm.all_keys()
    rng = np.random.default_rng(1)
    n = BATCH
    metas = [bytes([i]) * 16 for i in range(16)]
    dmeta = torch.from_numpy(np.frombuffer(b"".join(metas[i % 16] for i in range(n)), np.uint8).copy()).cuda()
    doff = torch.arange(0, 16 * (n + 1), 16, dtype=torch.int64, device="cuda")
    st = torch.empty((n,), dtype=torch.uint8, device="cuda")
    for bits, pname, bname in SIZES:
        k, kb = pkeys[pname], bkeys[bname]
        assert k.n.bit_length() == bits == kb.n.bit_length()
        kl = k.klen
        line = {}
        c = torch.from_numpy(rng.integers(0, 256, size=(n, kl), dtype=np.uint8)).cuda()
        c[:, 0] = 0  # below N
        sig = torch.empty_like(c)
        key = [_be(k.n), _be(k.p), _be(k.q), _be(pow(k.q, -1, k.p))]
        kargs = [x for f in key for x in (f, len(f))]

        def pb_sign():
            check(L.cb200_pbrsa_blind_sign(*kargs, c.data_ptr(), dmeta.data_ptr(), doff.data_ptr(), sig.data_ptr(),
                                           st.data_ptr(), n))
        put(line, "pbrsa_blind_sign", [n / timed(pb_sign, a.steps, a.warmup) * 1e3 for _ in range(a.repeats)])
        assert not st.any().item()
        dp, dq, qinv = kb.crt()
        bargs = [x for f in (_be(kb.n), _be(kb.e), _be(kb.p), _be(kb.q), _be(dp), _be(dq), _be(qinv))
                 for x in (f, len(f))]

        def b_sign():
            check(L.cb200_brsa_blind_sign(*bargs, c.data_ptr(), sig.data_ptr(), st.data_ptr(), n))
        put(line, "brsa_blind_sign", [n / timed(b_sign, a.steps, a.warmup) * 1e3 for _ in range(a.repeats)])
        assert not st.any().item()
        # Verify: 256 signatures per scheme over 64-byte messages, repeated over the batch
        msgs = [rng.integers(0, 256, size=64, dtype=np.uint8).tobytes() for _ in range(256)]
        dm = torch.from_numpy(np.frombuffer(b"".join(msgs) * (n // 256), np.uint8).copy()).cuda()
        moff = torch.arange(0, 64 * (n + 1), 64, dtype=torch.int64, device="cuda")
        prng = __import__("random").Random(bits)
        psigs = [pm.sign(k, msgs[i], metas[i % 16], prng) for i in range(256)]
        pv = torch.from_numpy(np.tile(np.frombuffer(b"".join(psigs), np.uint8).reshape(256, kl), (n // 256, 1))).cuda()
        bsigs = [bm.raw_sign(kb, bm.os2ip(bm.emsa_pss_encode(m, bits - 1, bytes(48)))) for m in msgs]
        bv = torch.from_numpy(np.tile(np.frombuffer(b"".join(bsigs), np.uint8).reshape(256, kl), (n // 256, 1))).cuda()
        nb = _be(kb.n)
        eb = _be(kb.e)

        def pb_verify():
            check(L.cb200_pbrsa_verify(key[0], len(key[0]), dm.data_ptr(), moff.data_ptr(), dmeta.data_ptr(),
                                       doff.data_ptr(), pv.data_ptr(), st.data_ptr(), n))
        put(line, "pbrsa_verify", [n / timed(pb_verify, a.steps, a.warmup) * 1e3 for _ in range(a.repeats)])
        assert not st.any().item()

        def b_verify():
            check(L.cb200_brsa_verify(0, nb, len(nb), eb, len(eb), dm.data_ptr(), moff.data_ptr(), bv.data_ptr(),
                                      st.data_ptr(), n))
        put(line, "brsa_verify", [n / timed(b_verify, a.steps, a.warmup) * 1e3 for _ in range(a.repeats)])
        assert not st.any().item()
        line["brsa_over_pbrsa_sign"] = round(line["brsa_blind_sign_per_s"] / line["pbrsa_blind_sign_per_s"], 2)
        line["brsa_over_pbrsa_verify"] = round(line["brsa_verify_per_s"] / line["pbrsa_verify_per_s"], 2)
        res[f"rsa{bits}"] = line
    circl_b200.shutdown()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
