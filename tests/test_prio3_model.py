"""tests/prio3_model.py against the reference's Prio3 vectors (vdaf/prio3/testdata, copied as tests/golden/prio3_*):
every field of all 14 files for every aggregator (public share, input shares, prep shares, prep messages, out shares,
agg shares and the aggregate result) and the TurboSHAKE128 XOF vectors.  CPU only."""
import pytest

import prio3_model as M
from conftest import load_golden


def test_roots_of_unity():
    for F in (M.F64, M.F128):
        assert pow(F.root(F.k), 1 << F.k, F.p) == 1 and pow(F.root(F.k), 1 << (F.k - 1), F.p) != 1
    # the reference's largest roots, converted out of its Montgomery form (arith/fp64/fp.go, arith/fp128/fp.go)
    assert M.F64.root(32) == 0xda58878b0d514e98 * pow(2**64, -1, M.F64.p) % M.F64.p
    assert M.F128.root(32) == ((0xe0312b455090dc3d << 64) | 0x488a61cbe76f8796) * pow(2**128, -1, M.F128.p) % M.F128.p


def test_xof_vectors():
    x = load_golden("prio3_XofTurboShake128.json.gz")
    dst, seed, binder = (bytes.fromhex(x[k]) for k in ("dst", "seed", "binder"))

    def xof():
        return M.TurboShake128(1).write(len(dst).to_bytes(2, "little") + dst + bytes([M.SEED]) + seed + binder)
    assert xof().read(32).hex() == x["derived_seed"]
    P = M.Prio3(M.Histogram(1, 1), 2)
    assert M.F128.enc(P.vec(xof(), x["length"])).hex() == x["expanded_vec_field128"]


@pytest.mark.parametrize("name", M.VECTOR_FILES)
def test_vector_file(name):
    v = load_golden("prio3_%s.json.gz" % name)
    P = M.from_vector(name, v)
    vk = bytes.fromhex(v["verify_key"])
    outs = [[] for _ in range(P.shares)]
    for r in v["prep"]:
        nonce = bytes.fromhex(r["nonce"])
        pub, ins = P.shard(r["measurement"], nonce, bytes.fromhex(r["rand"]))
        assert pub.hex() == r["public_share"]
        assert [i.hex() for i in ins] == r["input_shares"]
        states, shares = [], []
        for a in range(P.shares):
            st, state, share = P.prep_init(vk, a, nonce, pub, ins[a])
            assert st == 0
            states.append(state)
            shares.append(share)
        assert [s.hex() for s in shares] == r["prep_shares"][0]
        st, msg = P.prep_shares_to_prep(shares)
        assert st == 0 and msg.hex() == r["prep_messages"][0]
        for a in range(P.shares):
            st, out = P.prep_next(states[a], msg)
            assert st == 0 and out.hex() == "".join(r["out_shares"][a])
            outs[a].append(out)
    agg = [P.aggregate(o) for o in outs]
    assert [a.hex() for a in agg] == v["agg_shares"]
    assert P.unshard(agg, len(v["prep"])) == v["agg_result"]
