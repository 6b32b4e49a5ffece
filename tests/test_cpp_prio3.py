"""The C++ circl::prio3 mirror (include/circl_b200.hpp) through tests/cpp/test_prio3.cpp: it compiles and links; on
the CPU, the wire sizes of every vector file's configuration and every configuration error; on the GPU, every vector
file through the per-report calls (PrepInit for each aggregator, PrepSharesToPrep, PrepNext, AggregateUpdate, Unshard),
and a tampered proof failing PrepSharesToPrep with ErrProofVerify."""
import os
import subprocess

import pytest

import prio3_model as M
from conftest import load_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def run(tmp_path_factory):
    from circl_b200 import _ffi
    _ffi.lib()
    path = str(tmp_path_factory.mktemp("prio3_cpp") / "test_prio3")
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "cpp", "test_prio3.cpp"), "-o", path,
           "-L", os.path.join(ROOT, "circl_b200"), "-lcirclb200", "-Wl,-rpath," + os.path.join(ROOT, "circl_b200")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr

    def go(lines):
        out = subprocess.run([path], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stderr
        res = out.stdout.splitlines()
        assert len(res) == len(lines), out.stdout
        return res
    return go


def _cfg(v, name):
    kind = {"Count": 1, "Sum": 2, "SumVec": 3, "Histogram": 4, "MultihotCountVec": 5}[name.split("_")[0]]
    return " ".join(str(x) for x in (kind, v["shares"], v.get("max_measurement", 0), v.get("length", 0),
                                     v.get("bits", 0), v.get("chunk_length", 0), v.get("max_weight", 0))) + \
        " " + (v["ctx"] or "-")


def test_sizes_and_errors(run):
    lines, want = [], []
    for name in M.VECTOR_FILES:
        v = load_golden("prio3_%s.json.gz" % name)
        z = M.from_vector(name, v).sizes()
        lines.append("sizes " + _cfg(v, name))
        want.append(" ".join(str(z[k]) for k in ("input_share_leader", "input_share_helper", "public_share",
                                                 "prep_share", "prep_msg", "prep_state", "out_share", "agg_share")))
    bad = ["1 1 0 0 0 0 0 -", "2 2 9223372036854775808 0 0 0 0 -", "3 2 0 1 65 1 0 -", "3 2 0 0 1 1 0 -",
           "4 2 0 3 0 0 0 -", "5 2 0 3 0 1 4 -", "4 2 0 4294967306 0 4294967306 0 -", "6 2 0 0 0 0 0 -"]
    lines += ["sizes " + b for b in bad]
    got = run(lines)
    assert got[:len(want)] == want
    assert all(g.startswith("ERR ") for g in got[len(want):])


def test_without_a_device_or_on_one(run):
    v = load_golden("prio3_Count_0.json.gz")
    p = v["prep"][0]
    got = run([f"next {_cfg(v, 'Count_0')} {''.join(p['out_shares'][0])} -"])
    assert got[0] == "NODEV" or got[0] == "0 " + "".join(p["out_shares"][0])


@pytest.mark.gpu
@pytest.mark.parametrize("name", M.VECTOR_FILES)
def test_vectors(run, name):
    v = load_golden("prio3_%s.json.gz" % name)
    P = M.from_vector(name, v)
    cfg = _cfg(v, name)
    lines = []
    for r in v["prep"]:
        for a in range(P.shares):
            lines.append(f"init {cfg} {v['verify_key']} {a} {r['nonce']} {r['public_share'] or '-'} "
                         f"{r['input_shares'][a]}")
        lines.append(f"decide {cfg} " + " ".join(r["prep_shares"][0]))
    got = run(lines)
    i = 0
    for r in v["prep"]:
        for a in range(P.shares):
            st, state, share = got[i].split()
            assert st == "0" and share == r["prep_shares"][0][a]
            nxt = run([f"next {cfg} {state} {r['prep_messages'][0] or '-'}"])[0]
            assert nxt == "0 " + "".join(r["out_shares"][a])
            i += 1
        assert got[i] == "0 " + (r["prep_messages"][0] or "-")
        i += 1
    res = run([f"unshard {cfg} {len(v['prep'])} " + " ".join(v["agg_shares"])])[0].split()
    want = v["agg_result"] if isinstance(v["agg_result"], list) else [v["agg_result"]]
    assert [int(x) for x in res] == want
    # a tampered proof share fails Decide
    shares = list(v["prep"][0]["prep_shares"][0])
    b = bytearray(bytes.fromhex(shares[0]))
    b[0] ^= 1
    shares[0] = b.hex()
    assert run([f"decide {cfg} " + " ".join(shares)])[0] == "8 prio3: ErrProofVerify"
