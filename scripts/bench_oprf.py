"""OPRF server rates (RFC 9497, suites P256-SHA256, P384-SHA384, P521-SHA512) on one GPU, device-resident: Evaluate
(m = 1, one shared key) and FullEvaluate (16-byte inputs) in each mode, with the curve's ECDH Shared of the same run as
the yardstick.  2^18 requests for P-256 and P-384, 2^16 for P-521; CUDA events around `steps` calls after `warmup`
calls, repeated `repeats` times: each rate is the median of the repeats, with their minimum and maximum beside it
(`*_spread`).  Prints one JSON object with the card name and its power limit, read in the same run.

  python scripts/bench_oprf.py [--steps 5] [--warmup 2] [--repeats 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SUITES = [("P256-SHA256", 32, 1 << 18, "cb200_p256"), ("P384-SHA384", 48, 1 << 18, "cb200_p384"),
          ("P521-SHA512", 66, 1 << 16, "cb200_p521")]


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


def rate(line, name, fn, n, a):
    """line[name + "_per_s"] = the median rate over the repeats, line[name + "_spread"] = [min, max]."""
    rs = sorted(n / timed(fn, a.steps, a.warmup) * 1e3 for _ in range(a.repeats))
    line[name + "_per_s"] = round(rs[len(rs) // 2])
    line[name + "_spread"] = [round(rs[0]), round(rs[-1])]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    import circl_b200
    from circl_b200 import oprf
    from circl_b200._ffi import check, lib
    circl_b200.init(0)
    L = lib()
    check(L.cb200_set_stream(torch.cuda.current_stream().cuda_stream))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=30).stdout.strip().splitlines()
    res = {"card": q[0] if q else "unknown", "m": 1, "input_bytes": 16, "steps": a.steps, "warmup": a.warmup,
           "repeats": a.repeats}
    rng = np.random.default_rng(1)
    for ident, ns, n, ecdh in SUITES:
        S = oprf.GetSuite(ident)
        key = oprf.DeriveKey(S, 0, bytes(32), b"bench")
        pk = key.Public().MarshalBinary()
        sk = torch.from_numpy(np.frombuffer(key.k, dtype=np.uint8).copy()).cuda()
        # blinded elements: [x_i] pk for random x_i, from a base-mode Evaluate of pk under per-op keys x_i
        xs = torch.from_numpy(rng.integers(0, 256, size=(n, ns), dtype=np.uint8)).cuda()
        xs[:, 0] = 0
        pkrows = torch.from_numpy(np.frombuffer(pk, dtype=np.uint8).copy()).cuda().repeat(n, 1)
        rnd = xs.clone()
        rnd[:, -1] |= 1
        st = torch.empty((n,), dtype=torch.uint8, device="cuda")
        blinded, _ = oprf.EvaluateBatch(S, 0, xs, pkrows, 1)  # rows [x_i] pk: valid elements
        ev = torch.empty_like(blinded)
        proof = torch.empty((n, 2 * ns), dtype=torch.uint8, device="cuda")
        inputs = torch.from_numpy(rng.integers(0, 256, size=n * 16, dtype=np.uint8)).cuda()
        off = torch.arange(0, 16 * (n + 1), 16, dtype=torch.int64, device="cuda")
        out = torch.empty((n, S.Nh), dtype=torch.uint8, device="cuda")
        info = b"bench info"
        line = {"requests": n}
        for mode in (0, 1, 2):
            ib, il = (info, len(info)) if mode == 2 else (None, 0)

            def ev_call():
                check(L.cb200_oprf_evaluate(S.id, mode, sk.data_ptr(), 0, blinded.data_ptr(), 1, rnd.data_ptr(), ib, il,
                                            ev.data_ptr(), proof.data_ptr(), st.data_ptr(), n))

            def full_call():
                check(L.cb200_oprf_full_evaluate(S.id, mode, sk.data_ptr(), 0, inputs.data_ptr(), off.data_ptr(), ib, il,
                                                 out.data_ptr(), st.data_ptr(), n))
            rate(line, f"evaluate_mode{mode}", ev_call, n, a)
            assert not st.any().item()
            rate(line, f"full_evaluate_mode{mode}", full_call, n, a)
            assert not st.any().item()
        # the yardstick: ECDH Shared of the same curve, per-op scalars, one point
        pts = torch.from_numpy(rng.integers(0, 256, size=(n, 1 + 2 * ns), dtype=np.uint8)).cuda()
        g = circl_b200_point(L, ecdh, ns)
        pts[:] = torch.from_numpy(g).cuda()
        sh = torch.empty((n, ns), dtype=torch.uint8, device="cuda")
        rate(line, "ecdh_shared", lambda: check(getattr(L, ecdh)(rnd.data_ptr(), pts.data_ptr(), sh.data_ptr(),
                                                                 st.data_ptr(), n)), n, a)
        line["ecdh_over_verifiable_evaluate"] = round(line["ecdh_shared_per_s"] / line["evaluate_mode1_per_s"], 2)
        res[ident] = line
    circl_b200.shutdown()
    print(json.dumps(res))


def circl_b200_point(L, ecdh, ns):
    """An uncompressed public point (KeyGen of scalar 7) for the ECDH yardstick."""
    k = np.zeros((1, ns), dtype=np.uint8)
    k[0, -1] = 7
    out = np.zeros((1, 1 + 2 * ns), dtype=np.uint8)
    from circl_b200._ffi import check
    check(getattr(L, ecdh)(k.ctypes.data, None, out.ctypes.data, None, 1))
    return out[0]


if __name__ == "__main__":
    main()
