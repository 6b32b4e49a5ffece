"""Prio3 aggregator rates (draft-irtf-cfrg-vdaf-14) on one GPU, device-resident: reports/s of PrepInit as the leader
and as a helper, PrepSharesToPrep, and PrepNext followed by Aggregate, for two shares and these configurations:
Count; Sum with max 2^16 - 1; Histogram of length 100 / chunk 10 and of length 10^4 / chunk 100; SumVec of length 1000
/ bits 8 / chunk 90 (about the square root of the 8000 measurement elements; the reference's own tests use chunk 3 on
length 4); MultiHotCountVec of length 100 / weight 10 / chunk 10.

Each batch repeats one valid report made by tests/prio3_model.py (the work of a report does not depend on its values,
apart from the XOF's rejections, which occur with probability about 2^-32 per Field64 element and 2^-59 per Field128
element).  CUDA events around `steps` calls after `warmup` calls, repeated `repeats` times: each rate is the median of
the repeats, with their minimum and maximum beside it (`*_spread`).

It also reports the TurboSHAKE128 permutations each report needs at each step (Keccak-p[1600,12] calls, from the
message and output lengths), the device's Keccak-p[1600,12] rate measured in the same run with cb200_keccak_f1600
(turbo = 1) on 2^22 states, and each step's share of that Keccak floor.  Prints one JSON object with the card name and
its power limit, read in the same run.

  python scripts/bench_prio3.py [--steps 5] [--warmup 2] [--repeats 5]
"""
import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "tests"))

import prio3_model as M  # noqa: E402

CTX = b"bench"
CONFIGS = [
    ("count", lambda: M.Count(), 1 << 18, lambda: 1),
    ("sum_65535", lambda: M.Sum(2**16 - 1), 1 << 18, lambda: 12345),
    ("histogram_100_10", lambda: M.Histogram(100, 10), 1 << 16, lambda: 42),
    ("histogram_10000_100", lambda: M.Histogram(10000, 100), 1 << 12, lambda: 4242),
    ("sumvec_1000_8_90", lambda: M.SumVec(1000, 8, 90), 1 << 12, lambda: [i % 256 for i in range(1000)]),
    ("mhcv_100_10_10", lambda: M.MultiHotCountVec(100, 10, 10), 1 << 16, lambda: [i % 11 == 0 for i in range(100)]),
]


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
    return rs[len(rs) // 2]


def perms(absorb, out):
    """Keccak-p[1600,12] calls of one TurboSHAKE128 use: absorb bytes of input, out bytes of output"""
    return math.ceil((absorb + 1) / 168) + max(0, math.ceil(out / 168) - 1)


def blocks(P):
    """TurboSHAKE128 permutations per report: (leader PrepInit, helper PrepInit, PrepSharesToPrep)"""
    c, F = P.c, P.F
    head = 2 + 8 + len(P.ctx) + 1 + M.SEED
    common = perms(head + 1 + M.NONCE, F.size * c.query_rand_len)
    if P.jr:
        common += perms(head + 1 + M.NONCE + F.size * c.meas_len, M.SEED)      # joint-rand part
        common += perms(head + M.SEED * P.shares, M.SEED)                     # corrected seed
        common += perms(head + 1, F.size * c.joint_rand_len)                  # joint randomness
    helper = perms(head + 1, F.size * c.meas_len) + perms(head + 2, F.size * c.proof_len)
    decide = perms(head + M.SEED * P.shares, M.SEED) if P.jr else 0
    return common, common + helper, decide


def u8(b, n):
    return torch.from_numpy(np.tile(np.frombuffer(b, np.uint8), (n, 1))).cuda() if b else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    import circl_b200
    from circl_b200 import prio3
    from circl_b200._ffi import check, lib
    circl_b200.init(0)
    L = lib()
    check(L.cb200_set_stream(torch.cuda.current_stream().cuda_stream))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=30).stdout.strip().splitlines()
    res = {"card": q[0] if q else "unknown", "shares": 2, "steps": a.steps, "warmup": a.warmup, "repeats": a.repeats}
    st = torch.randint(0, 2**62, (1 << 22, 25), dtype=torch.int64, device="cuda")
    kec = {}
    kps = rate(kec, "keccak_p1600_12", lambda: check(L.cb200_keccak_f1600(st.data_ptr(), st.shape[0], 1)),
               st.shape[0], a)
    res["keccak_p1600_12_per_s"], res["keccak_p1600_12_spread"] = kec["keccak_p1600_12_per_s"], \
        kec["keccak_p1600_12_spread"]
    del st
    rng = np.random.default_rng(5)
    res["configs"] = {}
    for name, mk, n, meas in CONFIGS:
        P = M.Prio3(mk(), 2, CTX)
        c = P.c
        V = {1: lambda: prio3.Count(2, CTX), 2: lambda: prio3.Sum(2, c.max, CTX),
             3: lambda: prio3.SumVec(2, c.length, c.bits, c.chunk, CTX),
             4: lambda: prio3.Histogram(2, c.length, c.chunk, CTX),
             5: lambda: prio3.MultiHotCountVec(2, c.length, 2**c.bits - 1 - c.offset, c.chunk, CTX)}[c.ID]()
        nonce = rng.bytes(16)
        vk = rng.bytes(32)
        pub, ins = P.shard(meas(), nonce, rng.bytes(P.rand_size()))
        N, PUB = u8(nonce, n), u8(pub, n)
        IN = [u8(ins[0], n), u8(ins[1], n)]
        outs = [V.PrepInitBatch(vk, ag, N, PUB, IN[ag]) for ag in (0, 1)]
        assert not any(o[2].any().item() for o in outs)
        rows = torch.cat([outs[0][1], outs[1][1]], dim=1).contiguous()
        msgs, dst = V.PrepSharesToPrepBatch(rows)
        assert not dst.any().item()
        line = {"reports": n, "meas_len": c.meas_len, "proof_len": c.proof_len, "calls": c.calls}
        bl = blocks(P)
        line["turboshake_perms_per_report"] = {"prep_init_leader": bl[0], "prep_init_helper": bl[1],
                                               "prep_shares_to_prep": bl[2]}
        r0 = rate(line, "prep_init_leader", lambda: V.PrepInitBatch(vk, 0, N, PUB, IN[0]), n, a)
        r1 = rate(line, "prep_init_helper", lambda: V.PrepInitBatch(vk, 1, N, PUB, IN[1]), n, a)
        r2 = rate(line, "prep_shares_to_prep", lambda: V.PrepSharesToPrepBatch(rows), n, a)
        M_ = msgs if msgs.shape[1] else None

        def next_agg():
            o, s = V.PrepNextBatch(outs[0][0], M_)
            V.AggregateBatch(o, s)
        rate(line, "prep_next_aggregate", next_agg, n, a)
        line["keccak_floor_share"] = {"prep_init_leader": round(r0 * bl[0] / kps, 4),
                                      "prep_init_helper": round(r1 * bl[1] / kps, 4),
                                      "prep_shares_to_prep": round(r2 * bl[2] / kps, 4)}
        res["configs"][name] = line
    print(json.dumps(res))
    circl_b200.shutdown()


if __name__ == "__main__":
    main()
