"""RSA blind-signature rates (RFC 9474, RSABSSA-SHA384) on one GPU, device-resident, at 2048, 3072 and 4096 bits under
one key each (the fixture keys of tests/golden/): BlindSign on random blinded messages and Verify (PSS, 48-byte salt)
of 64-byte messages.  CUDA events around `steps` calls after `warmup` calls, repeated `repeats` times: each rate is the
median of the repeats, with their minimum and maximum beside it (`*_spread`).

The yardstick is OpenSSL in the same run: RSA-PSS-SHA-384 signing and verification through the cryptography package
on every host core (one process per core, each timed over `--cpu-seconds`), repeated `repeats` times the same way.
Prints one JSON object with the card name and its power limit and the host's core count, read in the same run.

  python scripts/bench_brsa.py [--steps 3] [--warmup 1] [--repeats 5] [--cpu-seconds 1]
"""
import argparse
import concurrent.futures as cf
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

# (bits, fixture key, BlindSign batch, Verify batch)
SIZES = [(2048, "rsa2048", 1 << 16, 1 << 18), (3072, "rsa3072", 1 << 15, 1 << 17), (4096, "rsa4096", 1 << 14, 1 << 16)]


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


_KEY = None


def _openssl_worker(args):
    """ops per second of one core: sign (op 0) or verify (op 1) for `secs` seconds"""
    global _KEY
    nums, op, secs = args
    from cryptography.hazmat.primitives import hashes
    from cryptography.hazmat.primitives.asymmetric import padding, rsa
    n, e, d, p, q = nums
    if _KEY is None or _KEY.private_numbers().public_numbers.n != n:
        pub = rsa.RSAPublicNumbers(e, n)
        _KEY = rsa.RSAPrivateNumbers(p, q, d, d % (p - 1), d % (q - 1), pow(q, -1, p), pub).private_key()
    pad, h, msg = padding.PSS(padding.MGF1(hashes.SHA384()), 48), hashes.SHA384(), b"m" * 64
    sig = _KEY.sign(msg, pad, h)
    pk = _KEY.public_key()
    cnt, t0 = 0, time.perf_counter()
    while time.perf_counter() - t0 < secs:
        for _ in range(16):
            if op == 0:
                _KEY.sign(msg, pad, h)
            else:
                pk.verify(sig, msg, pad, h)
        cnt += 16
    return cnt / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--cpu-seconds", type=float, default=1.0)
    a = ap.parse_args()
    import brsa_model as bm
    import circl_b200
    from circl_b200 import blindrsa
    from circl_b200._ffi import check, lib
    circl_b200.init(0)
    L = lib()
    check(L.cb200_set_stream(torch.cuda.current_stream().cuda_stream))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=30).stdout.strip().splitlines()
    cores = os.cpu_count()
    res = {"card": q[0] if q else "unknown", "host_cores": cores, "steps": a.steps, "warmup": a.warmup,
           "repeats": a.repeats, "message_bytes": 64}
    keys = bm.all_keys()
    rng = np.random.default_rng(1)
    pool = cf.ProcessPoolExecutor(cores)
    for bits, name, ns, nv in SIZES:
        k = keys[name]
        assert k.n.bit_length() == bits
        kl = k.klen
        line = {"sign_batch": ns, "verify_batch": nv}
        signer = blindrsa.NewSigner(blindrsa.PrivateKey(k.n, k.e, k.d, [k.p, k.q]))
        args = []
        for f in signer._fields:
            args += [f, len(f)]
        c = torch.from_numpy(rng.integers(0, 256, size=(ns, kl), dtype=np.uint8)).cuda()
        c[:, 0] = 0  # below N
        sig = torch.empty_like(c)
        st = torch.empty((max(ns, nv),), dtype=torch.uint8, device="cuda")

        def sign_call():
            check(L.cb200_brsa_blind_sign(*args, c.data_ptr(), sig.data_ptr(), st.data_ptr(), ns))
        put(line, "blind_sign", [ns / timed(sign_call, a.steps, a.warmup) * 1e3 for _ in range(a.repeats)])
        assert not st[:ns].any().item()
        # Verify: PSS encodings of 64-byte messages, signed on the GPU, repeated over the batch
        msgs = [rng.integers(0, 256, size=64, dtype=np.uint8).tobytes() for _ in range(256)]
        ems = [bm.emsa_pss_encode(m, bits - 1, bytes(48)).rjust(kl, b"\0") for m in msgs]
        s256 = signer.BlindSignBatch(np.frombuffer(b"".join(ems), np.uint8).reshape(256, kl).copy())
        reps = nv // 256
        sv = torch.from_numpy(np.tile(s256, (reps, 1))).cuda()
        dm = torch.from_numpy(np.frombuffer(b"".join(msgs) * reps, np.uint8).copy()).cuda()
        off = torch.arange(0, 64 * (nv + 1), 64, dtype=torch.int64, device="cuda")
        n_, e_ = signer._fields[0], signer._fields[1]

        def verify_call():
            check(L.cb200_brsa_verify(0, n_, len(n_), e_, len(e_), dm.data_ptr(), off.data_ptr(), sv.data_ptr(),
                                      st.data_ptr(), nv))
        put(line, "verify", [nv / timed(verify_call, a.steps, a.warmup) * 1e3 for _ in range(a.repeats)])
        assert not st[:nv].any().item()
        nums = (k.n, k.e, k.d, k.p, k.q)
        for op, label in ((0, "openssl_sign"), (1, "openssl_verify")):
            put(line, label, [sum(pool.map(_openssl_worker, [(nums, op, a.cpu_seconds)] * cores))
                              for _ in range(a.repeats)])
        line["gpu_over_openssl_sign"] = round(line["blind_sign_per_s"] / line["openssl_sign_per_s"], 2)
        line["gpu_over_openssl_verify"] = round(line["verify_per_s"] / line["openssl_verify_per_s"], 2)
        res[f"rsa{bits}"] = line
    pool.shutdown()
    circl_b200.shutdown()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
