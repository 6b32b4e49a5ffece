"""CPU: the FrodoKEM-640-SHAKE oracle (oracle/frodo.c) and the numpy model (tests/frodo_model.py) each reproduce the
reference's PQCgenKAT transcript hash, and agree with each other on random seeds, on implicit rejection (a flipped bit
in the B' part and in the C part of a ciphertext), on private keys whose S holds arbitrary 16-bit values and on public
keys made of arbitrary bytes."""
import numpy as np
import pytest

import frodo_model as M
from conftest import load_golden


@pytest.fixture(scope="module")
def O():
    from oracle import frodo as oracle_frodo
    return oracle_frodo


@pytest.fixture(scope="module")
def kat():
    return load_golden("frodo_vectors.json.gz")["kats"][0]


def _lists(f):
    return lambda *cols: tuple(map(list, zip(*[f(*a) for a in zip(*cols)])))


def test_oracle_pqcgenkat(O, kat):
    assert M.kat_hash(_lists(O.keygen), _lists(O.encaps), lambda sks, cts: [O.decaps(s, c) for s, c in zip(sks, cts)],
                      name=kat["name"]) == kat["sha256"]


def test_model_pqcgenkat(kat):
    assert M.kat_hash(_lists(M.keygen), _lists(M.encaps), lambda sks, cts: [M.decaps(s, c) for s, c in zip(sks, cts)],
                      name=kat["name"]) == kat["sha256"]


def test_oracle_equals_model_random(O):
    rng = np.random.default_rng(5)
    for _ in range(4):
        seed, mu = rng.bytes(48), rng.bytes(16)
        pk, sk = O.keygen(seed)
        assert (pk, sk) == M.keygen(seed)
        ct, ss = O.encaps(pk, mu)
        assert (ct, ss) == M.encaps(pk, mu)
        assert O.decaps(sk, ct) == ss == M.decaps(sk, ct)
        for pos, bit in ((int(rng.integers(0, 9600)), 1), (9600 + int(rng.integers(0, 120)), 0x40)):
            bad = bytearray(ct)
            bad[pos] ^= bit
            r = O.decaps(sk, bytes(bad))
            assert r == M.decaps(sk, bytes(bad)) and r != ss
            assert r == M.shake(16, bytes(bad), sk[:16])  # F(ct || s)


def test_oracle_equals_model_arbitrary_keys(O):
    rng = np.random.default_rng(6)
    for _ in range(3):
        sk, pk, ct, mu = rng.bytes(19888), rng.bytes(9616), rng.bytes(9720), rng.bytes(16)
        assert O.decaps(sk, ct) == M.decaps(sk, ct)
        assert O.encaps(pk, mu) == M.encaps(pk, mu)
        # a real key pair with S replaced by arbitrary 16-bit values
        pk2, sk2 = O.keygen(rng.bytes(48))
        ct2, _ = O.encaps(pk2, mu)
        sk2 = sk2[:16 + 9616] + rng.bytes(10240) + sk2[-16:]
        assert O.decaps(sk2, ct2) == M.decaps(sk2, ct2)


def test_batch_entry_matches_single_calls(O):
    rng = np.random.default_rng(8)
    seeds = rng.integers(0, 256, size=(5, 48), dtype=np.uint8)
    pk, sk = O.keygen_batch(seeds, nthreads=3)
    assert (pk[4].tobytes(), sk[4].tobytes()) == O.keygen(seeds[4].tobytes())
    es = rng.integers(0, 256, size=(5, 16), dtype=np.uint8)
    ct, ss = O.encaps_batch(pk[1], es, nthreads=2)  # one shared key
    assert (ct[3].tobytes(), ss[3].tobytes()) == O.encaps(pk[1].tobytes(), es[3].tobytes())
    assert np.array_equal(O.decaps_batch(sk[1], ct, nthreads=4), ss)
