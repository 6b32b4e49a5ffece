"""circl_b200/csrc/prio3.cuh compiled for the host (g++, no GPU) through tests/cpp/test_prio3_host.cpp, against
tests/prio3_model.py and Python integers: Field64 / Field128 multiplication, addition, subtraction and inversion at 0, 1,
p - 1 and random values; the NTT and its inverse at every domain size up to 2^10; and PrepInit (XOF expansion, Query
with the Lagrange-weight wire checks and the NTT-evaluated gadget) and PrepSharesToPrep (Decide) for every aggregator
of every reference vector and for random reports, valid and invalid, at several parameter sets of each circuit; and
Query at injected points t, including every t = alpha^k of the domain, where t^p = 1 gives ErrInvalidEval."""
import os
import random
import subprocess

import pytest

import prio3_model as M
from conftest import load_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def run(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("prio3") / "prio3_host")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Wno-unknown-pragmas",
                        os.path.join(ROOT, "tests", "cpp", "test_prio3_host.cpp"), "-o", path],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]

    def go(lines):
        out = subprocess.run([path], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stderr
        res = out.stdout.splitlines()
        assert len(res) == len(lines)
        return res
    return go


def _h(F, x):
    return x.to_bytes(F.size, "big").hex()


def _x(b):
    return b.hex() if b else "-"


def cfg_line(P):
    c = P.c
    _, log2p = M.next_pow2(1 + c.calls)
    f = [c.ID, P.shares, c.meas_len, c.output_len, c.eval_output_len, c.proof_len, c.verifier_len, c.joint_rand_len,
         c.gadget.arity, c.calls, getattr(c, "chunk", 0), getattr(c, "bits", 0), getattr(c, "length", 0), log2p,
         getattr(c, "offset", 0)]
    return " ".join(str(v) for v in f) + " " + _x(P.ctx)


@pytest.mark.parametrize("F", [M.F64, M.F128], ids=["f64", "f128"])
def test_field_ops(run, F):
    p, rng = F.p, random.Random(F.size)
    edge = [0, 1, 2, p - 1, p - 2, (p - 1) // 2, 2**32 - 1, 2**32, 2**63] + \
        ([2**64 - 1, 2**64, 2**127] if F.size == 16 else [])
    vals = edge + [rng.randrange(p) for _ in range(12)]
    lines, want = [], []
    for a in vals:
        for b in vals:
            for op, v in (("fmul", a * b % p), ("fadd", (a + b) % p), ("fsub", (a - b) % p)):
                lines.append(f"{op} {F.size * 8} {_h(F, a)} {_h(F, b)}")
                want.append(_h(F, v))
        lines.append(f"finv {F.size * 8} {_h(F, a)} {_h(F, 0)}")
        want.append(_h(F, pow(a, p - 2, p)))
    assert run(lines) == want


@pytest.mark.parametrize("F", [M.F64, M.F128], ids=["f64", "f128"])
def test_ntt_round_trip(run, F):
    rng = random.Random(3 * F.size)
    lines, want = [], []
    for logn in range(0, 11):
        v = [rng.randrange(F.p) for _ in range(1 << logn)]
        lines.append(f"ntt {F.size * 8} {logn} " + " ".join(_h(F, x) for x in v))
        want.append(" ".join(_h(F, x) for x in F.ntt(v, 1 << logn) + v))
    assert run(lines) == want


def _reports(P, vk, rows):
    """PrepInit / PrepSharesToPrep lines for (nonce, public share, input shares) rows, and the model's answers"""
    cl = cfg_line(P)
    init_lines, init_want, dec_lines, dec_want = [], [], [], []
    for nonce, pub, ins in rows:
        shares = []
        for a in range(P.shares):
            st, state, share = P.prep_init(vk, a, nonce, pub, ins[a])
            init_lines.append(f"init {cl} {vk.hex()} {a} {nonce.hex()} {_x(pub)} {_x(ins[a])}")
            init_want.append(f"{st} {_x(state) if not st else '-'} {_x(share) if not st else '-'}")
            shares.append(share)
        st, msg = P.prep_shares_to_prep(shares)
        dec_lines.append(f"decide {cl} {b''.join(shares).hex()}")
        dec_want.append(f"{st} {_x(msg) if not st else '-'}")
    return init_lines + dec_lines, init_want + dec_want


@pytest.mark.parametrize("name", M.VECTOR_FILES)
def test_vector_prep(run, name):
    v = load_golden("prio3_%s.json.gz" % name)
    P = M.from_vector(name, v)
    rows = []
    for r in v["prep"]:
        nonce = bytes.fromhex(r["nonce"])
        rows.append((nonce, bytes.fromhex(r["public_share"]), [bytes.fromhex(s) for s in r["input_shares"]]))
    lines, want = _reports(P, bytes.fromhex(v["verify_key"]), rows)
    got = run(lines)
    assert got == want
    # and the reference's own prep shares and messages
    shares = [s for r in v["prep"] for s in r["prep_shares"][0]]
    assert [g.split()[2] for g in got if len(g.split()) == 3] == shares
    assert [g.split()[1] for g in got if len(g.split()) == 2] == [r["prep_messages"][0] or "-" for r in v["prep"]]


def _hot(rng, length, weight):
    on = set(rng.sample(range(length), weight))
    return [i in on for i in range(length)]


CONFIGS = [
    ("count", lambda s: M.Count(), lambda rng, c: rng.randrange(2)),
    ("sum0", lambda s: M.Sum(0), lambda rng, c: 0),
    ("sum", lambda s: M.Sum(1000), lambda rng, c: rng.randrange(1001)),
    ("sumvec", lambda s: M.SumVec(20, 3, 7), lambda rng, c: [rng.randrange(8) for _ in range(20)]),
    ("histogram", lambda s: M.Histogram(50, 7), lambda rng, c: rng.randrange(50)),
    ("mhcv", lambda s: M.MultiHotCountVec(13, 5, 4), lambda rng, c: _hot(rng, 13, rng.randrange(6))),
]


def _tamper(P, rng, nonce, pub, ins, how):
    F = P.F
    ins = list(ins)
    if how == "proof":  # one leader proof element changed
        off = F.size * (P.c.meas_len + rng.randrange(P.c.proof_len))
        x = (int.from_bytes(ins[0][off:off + F.size], "little") + 1) % F.p
        ins[0] = ins[0][:off] + x.to_bytes(F.size, "little") + ins[0][off + F.size:]
    elif how == "noncanonical":
        off = F.size * rng.randrange(P.c.meas_len + P.c.proof_len)
        ins[0] = ins[0][:off] + (F.p + rng.randrange(2**(8 * F.size) - F.p)).to_bytes(F.size, "little") + \
            ins[0][off + F.size:]
    elif how == "public" and pub:
        i = rng.randrange(len(pub))
        pub = pub[:i] + bytes([pub[i] ^ 1]) + pub[i + 1:]
    return nonce, pub, ins


@pytest.mark.parametrize("shares", [2, 3])
@pytest.mark.parametrize("name,mk,meas", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_random_reports(run, name, mk, meas, shares):
    rng = random.Random(name + str(shares))
    P = M.Prio3(mk(shares), shares, b"ctx" * shares)
    vk = rng.randbytes(32)
    rows = []
    for i in range(6):
        nonce = rng.randbytes(16)
        pub, ins = P.shard(meas(rng, P.c), nonce, rng.randbytes(P.rand_size()))
        rows.append(_tamper(P, rng, nonce, pub, ins, ["", "", "proof", "noncanonical", "public", ""][i]))
    lines, want = _reports(P, vk, rows)
    assert run(lines) == want
    assert any(w.startswith("8 ") for w in want)  # a tampered proof fails Decide


@pytest.mark.parametrize("name,mk,meas", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_query_at_injected_t(run, name, mk, meas):
    """ErrInvalidEval (status 4) cannot be produced through a verify key; inject t, including every alpha^k"""
    rng = random.Random("t" + name)
    P = M.Prio3(mk(2), 2, b"inject")
    c, F = P.c, P.F
    nonce = rng.randbytes(16)
    pub, ins = P.shard(meas(rng, c), nonce, rng.randbytes(P.rand_size()))
    nm = F.size * (c.meas_len + c.proof_len)
    meas_s, proof = F.dec(ins[0][:F.size * c.meas_len]), F.dec(ins[0][F.size * c.meas_len:nm])
    jr = []
    if P.jr:
        part = P.joint_rand_part(ins[0][nm:], 0, nonce, F.enc(meas_s))
        jr = P.joint_rands(P.joint_rand_seed(part + pub[M.SEED:]))
    p, log2p = M.next_pow2(1 + c.calls)
    alpha = F.root(log2p)
    ts = [pow(alpha, k, F.p) for k in range(p)] + [rng.randrange(F.p) for _ in range(4)] + [0]
    lines, want = [], []
    for t in ts:
        qr = [rng.randrange(F.p) for _ in range(c.query_rand_len)]
        qr[c.eval_output_len if c.eval_output_len > 1 else 0] = t
        ver = c.query(meas_s, proof, qr, jr, 2)
        lines.append(f"query {cfg_line(P)} {F.enc([t]).hex()} {_x(ins[0][:nm])} {_x(F.enc(jr))} {F.enc(qr).hex()}")
        want.append("4 -" if ver is None else f"0 {F.enc(ver).hex()}")
    assert run(lines) == want
    assert want[:p] == ["4 -"] * p and all(w.startswith("0 ") for w in want[p:])
