"""Threshold RSA on the GPU against tests/tssrsa_model.py and OpenSSL: signature shares under every fixture key at
(players, threshold) = (3, 2) and (64, 33), with edge digests, a cached twoDeltaSi that disagrees with s_i and CUDA
tensors; a deal-sign-combine round trip with a random index set per op, verified by OpenSSL for PKCS #1 v1.5 and PSS;
every failure class in one batch; e = 3 at players = 3 (gcd(e', e) = 3); device rows at odd byte offsets; and a host
batch past three staging chunks split across every visible GPU."""
import random

import numpy as np
import pytest

import brsa_model as bm
import tssrsa_model as tm
from test_tssrsa_host import edge_ops

pytestmark = pytest.mark.gpu
KEYS = ["rsa2048", "rsa3072", "rsa3073", "rsa2048e3", "rsa2048u", "rsa3000u", "rsa4096"]


@pytest.fixture(scope="module")
def cb():
    import circl_b200
    circl_b200.init(0)
    yield circl_b200
    circl_b200.shutdown()


class _Pub:
    def __init__(self, k):
        self.N, self.E = k.n, k.e


class _Stream:
    def __init__(self, rng):
        self.rng = rng

    def read(self, n):
        return self.rng.randbytes(n)


def _shares(k, players, threshold, rng):
    from circl_b200 import tssrsa
    key = type("K", (), {"E": k.e, "Primes": [k.p, k.q]})
    return tssrsa.Deal(_Stream(rng), players, threshold, key, False)


def _rows(vals, kl):
    return np.frombuffer(b"".join(v.to_bytes(kl, "big") for v in vals), np.uint8).reshape(len(vals), kl).copy()


def _ints(rows):
    rows = rows.cpu().numpy() if hasattr(rows, "cpu") else rows
    return [int.from_bytes(r.tobytes(), "big") for r in rows]


@pytest.mark.parametrize("players,threshold", [(3, 2), (64, 33)])
@pytest.mark.parametrize("name", KEYS)
def test_sign_shares_match_pow(cb, name, players, threshold):
    import torch
    k = bm.all_keys()[name]
    kl, pub = k.klen, _Pub(k)
    rng = random.Random(f"{name}{players}")
    ks = _shares(k, players, threshold, rng)
    assert [s.si for s in ks] == tm.deal(_Stream(random.Random(f"{name}{players}")), players, threshold, k.p, k.q,
                                         k.e)
    n = 1 << 12
    xs = [0, 1, k.n - 1, k.n, k.n + 1, (1 << (8 * kl)) - 1] + [rng.randrange(1 << (8 * kl)) for _ in range(n - 6)]
    rows = _rows(xs, kl)
    share = ks[-1]
    got = _ints(share.SignBatch(pub, rows))
    E = 2 * tm.delta(players) * share.si
    for i in list(range(8)) + list(range(8, n, 97)):
        assert got[i] == pow(xs[i], E, k.n), i
    dev = share.SignBatch(pub, torch.from_numpy(rows).cuda())
    assert _ints(dev) == got
    # a cached twoDeltaSi is used as given, even when it disagrees with s_i
    from circl_b200 import tssrsa
    odd = tssrsa.KeyShare(share.si, share.Index, players, threshold, twoDeltaSi=E + 12345)
    got = _ints(odd.SignBatch(pub, rows[:64]))
    assert got == [pow(x, E + 12345, k.n) for x in xs[:64]]
    # Sign reduces a digest longer than kLen bytes
    long = (k.n * 5 + 7).to_bytes(kl + 1, "big")
    assert share.Sign(None, pub, long, True).xi == pow(7, E, k.n)


@pytest.mark.parametrize("name", ["rsa2048", "rsa3073", "rsa4096"])
def test_round_trip_openssl(cb, name):
    from cryptography.hazmat.primitives import hashes
    from cryptography.hazmat.primitives.asymmetric import padding, rsa
    from circl_b200 import tssrsa
    k = bm.all_keys()[name]
    kl, pub = k.klen, _Pub(k)
    osk = rsa.RSAPrivateNumbers(k.p, k.q, k.d, k.d % (k.p - 1), k.d % (k.q - 1), pow(k.q, -1, k.p),
                                rsa.RSAPublicNumbers(k.e, k.n)).private_key()
    opk = osk.public_key()
    rng = random.Random(name)
    players, threshold = 7, 4
    ks = _shares(k, players, threshold, rng)
    cases = []
    for h, ch in (("sha256", hashes.SHA256()), ("sha384", hashes.SHA384())):
        for pss in (False, True):
            for m in (b"hello", rng.randbytes(100)):
                padder = tssrsa.PSSPadder(_Stream(rng)) if pss else tssrsa.PKCS1v15Padder()
                cases.append((h, ch, pss, m, tssrsa.PadHash(padder, h, pub, m)))
    n = len(cases)
    # every op its own index set of size threshold .. players
    sets = [sorted(rng.sample(range(1, players + 1), rng.randint(threshold, players))) for _ in range(n)]
    xs = [int.from_bytes(c[4], "big") for c in cases]
    shares = {j: _ints(ks[j - 1].SignBatch(pub, _rows(xs, kl))) for j in range(1, players + 1)}
    got = {}
    for size in sorted({len(s) for s in sets}):
        ops = [i for i in range(n) if len(sets[i]) == size]
        idx = np.array([sets[i] for i in ops], np.uint16)
        xi = np.stack([_rows([shares[j][i] for j in sets[i]], kl) for i in ops])
        sig = tssrsa.CombineSignSharesBatch(pub, players, threshold, idx, xi, _rows([xs[i] for i in ops], kl))
        for r, i in enumerate(ops):
            st, y = tm.combine(k.n, k.e, players, sets[i], [shares[j][i] for j in sets[i]], xs[i])
            assert st == 0 and int.from_bytes(sig[r].tobytes(), "big") == y
            got[i] = sig[r].tobytes()
            h, ch, pss, m, _ = cases[i]
            if pss:
                opk.verify(sig[r].tobytes(), m, padding.PSS(padding.MGF1(ch), padding.PSS.AUTO), ch)
            else:
                opk.verify(sig[r].tobytes(), m, padding.PKCS1v15(), ch)
                assert sig[r].tobytes() == osk.sign(m, padding.PKCS1v15(), ch)  # the root is unique
    # the single-op form, and the reference's parameter errors before any served-range rule
    sh = [tssrsa.SignShare(shares[j][0], j, players, threshold) for j in sets[0]]
    assert tssrsa.CombineSignShares(pub, players, threshold, sh, cases[0][4]) == got[0]
    with pytest.raises(ValueError, match="insufficient shares"):
        tssrsa.CombineSignShares(pub, players, threshold, sh[:threshold - 1], cases[0][4])
    with pytest.raises(tssrsa.ErrInvalidCalc):
        tssrsa.CombineSignShares(pub, players, threshold, [tssrsa.SignShare(1, 0, players, threshold)] + sh,
                                 cases[0][4])


def _combine_batch(k, players, threshold, ops, dev=False):
    import torch
    from circl_b200 import tssrsa
    kl = k.klen
    kk = len(ops[0][0])
    idx = np.array([o[0] for o in ops], np.uint16)
    xi = np.stack([_rows(o[1], kl) for o in ops]).reshape(len(ops), kk * kl)
    msgs = _rows([o[2] for o in ops], kl)
    if dev:
        idx = torch.from_numpy(idx.view(np.int16)).cuda()
        xi, msgs = torch.from_numpy(xi).cuda(), torch.from_numpy(msgs).cuda()
    try:
        sig = tssrsa.CombineSignSharesBatch(_Pub(k), players, threshold, idx, xi, msgs)
        st = np.zeros(len(ops), np.uint8)
    except tssrsa.TSSRSAError as err:
        sig, st = err.results, err.status
    if dev:
        sig = sig.cpu().numpy()
        st = st.cpu().numpy() if hasattr(st, "cpu") else st
    return _ints(sig), list(st)


@pytest.mark.parametrize("name,players,threshold", [("rsa2048", 3, 2), ("rsa3073", 3, 2), ("rsa2048", 7, 4),
                                                    ("rsa4096", 5, 3)])
def test_failure_classes_in_one_batch(cb, name, players, threshold):
    k = bm.all_keys()[name]
    rng = random.Random(name + "f")
    ops = edge_ops(k, players, threshold, rng)
    want = [tm.combine(k.n, k.e, players, *o) for o in ops]
    for size in sorted({len(o[0]) for o in ops}):
        sel = [i for i, o in enumerate(ops) if len(o[0]) == size]
        for dev in (False, True):
            y, st = _combine_batch(k, players, threshold, [ops[i] for i in sel], dev)
            assert [(int(s), v) for s, v in zip(st, y)] == [want[i] for i in sel]
    assert {w[0] for w in want} == {0, 1, 2}


def test_e3_at_three_players(cb):
    k = bm.all_keys()["rsa2048e3"]
    rng = random.Random("e3")
    s = _shares(k, 3, 2, rng)
    E = [2 * tm.delta(3) * v.si for v in s]
    xs = [rng.randrange(k.n) for _ in range(30)] + [0, 1]
    ops = [([1, 2], [pow(x, E[0], k.n), pow(x, E[1], k.n)], x) for x in xs]
    y, st = _combine_batch(k, 3, 2, ops)
    want = [tm.combine(k.n, k.e, 3, *o) for o in ops]
    assert [(int(a), b) for a, b in zip(st, y)] == want
    assert all(w[0] == 2 for w in want[:-2]) and want[-2] == (0, 0) and want[-1] == (0, 1)


def test_device_rows_at_odd_offsets_and_misaligned_idx(cb):
    import torch
    from circl_b200 import _ffi
    k = bm.all_keys()["rsa2048"]
    kl, n, players = k.klen, 40, 3
    rng = random.Random("odd")
    s = _shares(k, players, 2, rng)
    E = [2 * tm.delta(players) * v.si for v in s]
    xs = [rng.randrange(k.n) for _ in range(n)]
    L = _ffi.lib()
    nb, eb = bm.i2osp(k.n, kl), bm.i2osp(k.e, 3)
    buf = torch.zeros(2 * n * kl + 8, dtype=torch.uint8, device="cuda")
    din = buf[1:1 + n * kl]
    din.copy_(torch.from_numpy(_rows(xs, kl).reshape(-1)))
    dout = buf[n * kl + 3:n * kl + 3 + n * kl]
    tds = bm.i2osp(E[0], (E[0].bit_length() + 7) // 8)
    _ffi.check(L.cb200_tssrsa_sign_share(nb, len(nb), players, tds, len(tds), din.data_ptr(), dout.data_ptr(), n))
    torch.cuda.synchronize()
    assert _ints(dout.cpu().numpy().reshape(n, kl)) == [pow(x, E[0], k.n) for x in xs]
    # combine with every row buffer at an odd offset, idx 2-byte aligned
    x1 = [pow(x, E[0], k.n) for x in xs]
    x2 = [pow(x, E[1], k.n) for x in xs]
    xi = np.concatenate([_rows(x1, kl), _rows(x2, kl)], axis=1)
    big = torch.zeros(4 * n * kl + 64, dtype=torch.uint8, device="cuda")
    dxi = big[1:1 + 2 * n * kl]
    dxi.copy_(torch.from_numpy(xi.reshape(-1)))
    dm = big[2 * n * kl + 3:3 * n * kl + 3]
    dm.copy_(torch.from_numpy(_rows(xs, kl).reshape(-1)))
    dsig = big[3 * n * kl + 5:4 * n * kl + 5]
    dst = torch.zeros(n + 1, dtype=torch.uint8, device="cuda")[1:]
    idx = torch.from_numpy(np.array([[1, 2]] * n, np.int16)).cuda()
    _ffi.check(L.cb200_tssrsa_combine(nb, len(nb), eb, len(eb), players, 2, 2, idx.data_ptr(), dxi.data_ptr(),
                                      dm.data_ptr(), dsig.data_ptr(), dst.data_ptr(), n))
    torch.cuda.synchronize()
    assert not dst.cpu().numpy().any()
    assert _ints(dsig.cpu().numpy().reshape(n, kl)) == [tm.combine(k.n, k.e, players, [1, 2], [a, b], x)[1]
                                                         for a, b, x in zip(x1, x2, xs)]
    rc = L.cb200_tssrsa_combine(nb, len(nb), eb, len(eb), players, 2, 2, idx.data_ptr() + 1, dxi.data_ptr(),
                                dm.data_ptr(), dsig.data_ptr(), dst.data_ptr(), n)
    with pytest.raises(_ffi.Cb200Error):
        _ffi.check(rc)


def test_host_batch_past_three_chunks_on_every_gpu():
    import circl_b200
    from circl_b200 import tssrsa
    circl_b200.init_devices(0)  # every visible GPU; with one, the batch still crosses staging chunks
    try:
        k = bm.all_keys()["rsa2048"]
        kl, players, threshold = k.klen, 64, 33
        rng = random.Random("chunks")
        s = _shares(k, players, threshold, rng)
        kk = 64
        row = kk * kl + 2 * kk + kl + 1
        chunk = (64 << 20) // row
        n = 3 * chunk + 1000  # several staging chunks and, with more than one GPU, several shards
        # 16 distinct ops, tiled: the shares come from the GPU, one SignBatch per party
        base = 16
        xs = [rng.randrange(k.n) for _ in range(base)]
        sets = [rng.sample(range(1, players + 1), kk) for _ in range(base)]
        sh = {j: _ints(s[j - 1].SignBatch(_Pub(k), _rows(xs, kl))) for j in range(1, players + 1)}
        xi = np.stack([_rows([sh[j][i] for j in sets[i]], kl).reshape(-1) for i in range(base)])
        xi[3, 5] ^= 1  # one corrupted op in the tile
        reps = -(-n // base)
        idx = np.tile(np.array(sets, np.uint16), (reps, 1))[:n]
        xin = np.tile(xi, (reps, 1))[:n]
        msgs = np.tile(_rows(xs, kl), (reps, 1))[:n]
        with pytest.raises(tssrsa.ErrInternal) as ei:
            tssrsa.CombineSignSharesBatch(_Pub(k), players, threshold, idx, xin, msgs)
        st, sig = ei.value.status, ei.value.results
        want = []
        for i in range(base):
            xv = [int.from_bytes(xi[i, t * kl:(t + 1) * kl].tobytes(), "big") for t in range(kk)]
            want.append(tm.combine(k.n, k.e, players, sets[i], xv, xs[i]))
        y = _ints(sig)
        for i in range(n):
            assert (int(st[i]), y[i]) == want[i % base], i
    finally:
        circl_b200.shutdown()
