"""Every kernel family of the library once, at small sizes, for compute-sanitizer (scripts/sanitize_r02.sh):
memcheck / racecheck / synccheck / initcheck need short runs.  Results are still checked against the oracle."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import circl_b200  # noqa: E402
import oracle
from circl_b200 import dilithium, hybrid, keccak, kyber, mldsa, mlkem

circl_b200.init(0)
rng = np.random.default_rng(7)
Q = 3329

# raw ring kernels: the forward NTT stages its input with bulk-async (TMA) copies, one mbarrier per octet; both
# directions are run on in-contract inputs (fast path) and on arbitrary int16 (general path)
p = rng.integers(-Q, Q, size=(203, 256), dtype=np.int64).astype(np.int16)
assert np.array_equal(kyber.ntt_(p.copy()), oracle.kyber_ntt(p))
assert np.array_equal(kyber.inv_ntt_(p.copy()), oracle.kyber_invntt(p))
pa = rng.integers(-32768, 32768, size=(203, 256), dtype=np.int64).astype(np.int16)
assert np.array_equal(kyber.ntt_(pa.copy()), oracle.kyber_ntt(pa))
assert np.array_equal(kyber.inv_ntt_(pa.copy()), oracle.kyber_invntt(pa))
a = rng.integers(-Q, Q, size=(40, 3, 256), dtype=np.int64).astype(np.int16)
assert np.array_equal(kyber.poly_dot_hat(a, a, 3), oracle.kyber_dot(a, a, 3))
d = rng.integers(0, 8380417, size=(77, 256), dtype=np.int64).astype(np.uint32)
assert np.array_equal(dilithium.ntt_(d.copy()), np.stack([oracle.dil_ntt(x) for x in d]))

# Keccak and the samplers on their own
st = rng.integers(0, 1 << 62, size=(130, 25), dtype=np.uint64)
assert keccak.permute_(st.copy())[129].tolist() == oracle.keccak_f1600([int(x) for x in st[129]])
seeds = rng.integers(0, 256, size=(300, 32), dtype=np.uint8)
xy = rng.integers(0, 4, size=(300, 2), dtype=np.uint8)
u = kyber.derive_uniform(seeds, xy)
assert np.array_equal(u[299], oracle.kyber_derive_uniform(seeds[299].tobytes(), int(xy[299, 0]), int(xy[299, 1])))
assert np.array_equal(kyber.derive_noise(seeds, xy[:, 0].copy(), 2)[5], oracle.kyber_derive_noise(seeds[5].tobytes(), int(xy[5, 0]), 2))

# ML-KEM: keygen, encaps (IDP.2A encrypt kernel with register prefetch), decaps, for every parameter set
for name, k in (("ML-KEM-512", 2), ("ML-KEM-768", 3), ("ML-KEM-1024", 4)):
    s = mlkem.ByName(name)
    ek, dk = s.DeriveKeyPairBatch(rng.integers(0, 256, size=(37, 64), dtype=np.uint8))
    m = rng.integers(0, 256, size=(37, 32), dtype=np.uint8)
    ct, ss = s.EncapsulateBatch(ek, m)
    wct, wss, _ = oracle.mlkem_encaps_batch(k, ek, m, nthreads=2)
    assert np.array_equal(ct, wct) and np.array_equal(ss, wss)
    assert np.array_equal(s.DecapsulateBatch(dk, ct), ss)

# ML-DSA-65 / 44: the rejection loop (w_kernel: bulk-async ring over the rows of A), verify, keygen
for name in ("ML-DSA-65", "ML-DSA-44"):
    s = mldsa.ByName(name)
    pk, sk = s.DeriveKeyBatch(rng.integers(0, 256, size=(24, 32), dtype=np.uint8))
    msgs = [bytes([i]) * (i + 3) for i in range(24)]
    sig = s.SignBatch(sk, msgs)
    mode = int(name[-2:])
    assert sig[7].tobytes() == oracle.mldsa_sign(mode, sk[7].tobytes(), msgs[7])[0]
    assert s.VerifyBatch(pk, msgs, sig).all()

# wire-side callers
xw = hybrid.ByName("X-Wing")
xpk, xsk = xw.DeriveKeyPairBatch(rng.integers(0, 256, size=(9, 32), dtype=np.uint8))
es = rng.integers(0, 256, size=(9, 64), dtype=np.uint8)
xct, xss = xw.EncapsulateBatch(xpk, es)
assert np.array_equal(xw.DecapsulateBatch(xsk, xct), xss)

# FrodoKEM-640-SHAKE at n = 33: every kernel of csrc/frodo.cu -- the per-op path (A staged through shared memory, the
# B' compare folded with __syncthreads_or), the shared-key path (A planes, the GEMM and its cross-CTA atomicOr on the
# compare flag), implicit rejection in the B' and C parts
from circl_b200 import frodo  # noqa: E402
from oracle import frodo as oracle_frodo  # noqa: E402
fk = frodo.Scheme()
fpk, fsk = fk.DeriveKeyPairBatch(rng.integers(0, 256, size=(33, 48), dtype=np.uint8))
fes = rng.integers(0, 256, size=(33, 16), dtype=np.uint8)
fct, fss = fk.EncapsulateBatch(fpk, fes)
fbad = fct.copy()
fbad[::3, 17] ^= 1
fbad[1::3, 9700] ^= 1
assert fk.DecapsulateBatch(fsk, fbad)[0].tobytes() == oracle_frodo.decaps(fsk[0].tobytes(), fbad[0].tobytes())
pk0, sk0 = fk.UnmarshalBinaryPublicKey(fpk[0].tobytes()), fk.UnmarshalBinaryPrivateKey(fsk[0].tobytes())
sct, sss = fk.EncapsulateBatch(pk0, fes)
assert (sct[32].tobytes(), sss[32].tobytes()) == oracle_frodo.encaps(fpk[0].tobytes(), fes[32].tobytes())
sct[::2, 40] ^= 4
assert fk.DecapsulateBatch(sk0, sct)[2].tobytes() == oracle_frodo.decaps(fsk[0].tobytes(), sct[2].tobytes())
circl_b200.shutdown()
print("sanitize_ops ok")
