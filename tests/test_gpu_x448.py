"""GPU parity for dh/x448: the RFC 7748 vectors (dh/x448/key_test.go), KeyGen against Shared with u = 5, the oracle
and OpenSSL, per-op status for low-order and non-canonical points, host and device pointers."""
import hashlib

import numpy as np
import pytest

from conftest import load_golden

pytestmark = pytest.mark.gpu

P = 2**448 - 2**224 - 1
BASE = bytes([5] + [0] * 55)


@pytest.fixture(scope="module")
def cb():
    import circl_b200
    circl_b200.init(0)
    yield circl_b200
    circl_b200.shutdown()


def _rows(items):
    return np.frombuffer(b"".join(items), dtype=np.uint8).reshape(len(items), -1)


def _h(tag, i, n=56):
    return hashlib.shake_256(bytes([tag]) + i.to_bytes(8, "little")).digest(n)


def test_rfc7748_one_batch_and_iterated(cb):
    from circl_b200 import x448
    xv = load_golden("x448_vectors.json.gz")
    kat = xv["rfc7748_kat"]
    out, ok = x448.x448_shared(_rows([bytes.fromhex(v["scalar"]) for v in kat]), _rows([bytes.fromhex(v["input"]) for v in kat]))
    assert ok.all()
    assert [out[i].tobytes().hex() for i in range(len(kat))] == [v["output"] for v in kat]
    for v in xv["rfc7748_times"]:  # key_test.go:53-79, 1 and 1000 times
        u = k = BASE
        for _ in range(v["times"]):
            r = x448.x448_shared(_rows([k]), _rows([u]))[0][0].tobytes()
            u, k = k, r
        assert k.hex() == v["key"]


def test_keygen_equals_shared_and_matches_oracle_and_openssl(cb):
    from oracle import x448 as ox
    from cryptography.hazmat.primitives.asymmetric.x448 import X448PrivateKey, X448PublicKey
    from circl_b200 import x448
    n = 3000
    ks = _rows([_h(1, i) for i in range(n)])
    pub = x448.x448_keygen(ks)
    shared, ok = x448.x448_shared(ks, _rows([BASE] * n))
    assert ok.all() and (pub == shared).all()
    ks2 = _rows([_h(2, i) for i in range(n)])
    s12, ok12 = x448.x448_shared(ks, x448.x448_keygen(ks2))
    s21, _ = x448.x448_shared(ks2, pub)
    assert ok12.all() and (s12 == s21).all()
    for i in range(0, n, 211):
        assert pub[i].tobytes() == ox.x448(ks[i].tobytes())[0]
        assert pub[i].tobytes() == X448PrivateKey.from_private_bytes(ks[i].tobytes()).public_key().public_bytes_raw()
        pub2 = X448PrivateKey.from_private_bytes(ks2[i].tobytes()).public_key().public_bytes_raw()
        assert s12[i].tobytes() == X448PrivateKey.from_private_bytes(ks[i].tobytes()).exchange(
            X448PublicKey.from_public_bytes(pub2))
    us = _rows([_h(3, i) for i in range(500)])
    out, ok = x448.x448_shared(ks[:500], us)
    assert ok.all()
    for i in range(0, 500, 37):
        assert out[i].tobytes() == ox.x448(ks[i].tobytes(), us[i].tobytes())[0]


def test_per_op_status_low_order_and_non_canonical(cb):
    from oracle import x448 as ox
    from circl_b200 import x448
    n = 300
    ks = _rows([_h(4, i) for i in range(n)])
    us = [_h(5, i) for i in range(n)]
    special = {17: 0, 18: 1, 19: P - 1, 20: P, 21: P + 1, 150: 2**448 - 1, 151: P + 5}
    for i, u in special.items():
        us[i] = u.to_bytes(56, "little")
    out, ok = x448.x448_shared(ks, _rows(us))
    low = {17, 18, 19, 20, 21}
    assert [i for i in range(n) if not ok[i]] == sorted(low)
    for i in range(n):
        if i in low:
            assert out[i].tobytes() == bytes(56)
        elif i in special or i % 29 == 0:
            assert (out[i].tobytes(), True) == ox.x448(ks[i].tobytes(), us[i])


def test_device_pointers(cb):
    import torch
    from oracle import x448 as ox
    from circl_b200 import x448
    n = 4096
    g = torch.Generator(device="cpu").manual_seed(5)
    k = torch.randint(0, 256, (n, 56), dtype=torch.uint8, generator=g).cuda()
    u = torch.randint(0, 256, (n, 56), dtype=torch.uint8, generator=g).cuda()
    u[100] = 0
    pub = x448.x448_keygen(k)
    out, ok = x448.x448_shared(k, u)
    torch.cuda.synchronize()
    assert pub.is_cuda and out.is_cuda
    okc = ok.cpu().numpy()
    assert not okc[100] and okc.sum() == n - 1 and not out[100].any()
    for i in (0, 1234, n - 1):
        assert pub[i].cpu().numpy().tobytes() == ox.x448(k[i].cpu().numpy().tobytes())[0]
        assert out[i].cpu().numpy().tobytes() == ox.x448(k[i].cpu().numpy().tobytes(), u[i].cpu().numpy().tobytes())[0]
    host = x448.x448_keygen(k.cpu().numpy())
    assert np.array_equal(host, pub.cpu().numpy())
