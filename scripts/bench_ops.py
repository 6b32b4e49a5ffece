"""Device-resident timings of the secondary entry points (CUDA events, >= 3 warm-ups, inputs > L2).
Writes one JSON object; the headline contract lives in bench.py."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import circl_b200
from circl_b200 import dilithium as dl, kyber, mlkem
import bench as B

circl_b200.init(0)
res = {}


def timed(fn, steps=5, warm=3):
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


def eddsa_lines(res):
    """Ed25519 and Ed25519-Dilithium2 through the C ABI, device-resident, 2^18 operations, per-op keys, 32-byte messages
    (plus Ed25519 Verify on 1 KiB messages), with X25519 KeyGen / Shared of the same run for comparison."""
    from circl_b200 import hybrid
    from circl_b200._ffi import check, lib
    L = lib()
    check(L.cb200_set_stream(torch.cuda.current_stream().cuda_stream))
    n = 1 << 18
    g = torch.Generator(device="cuda").manual_seed(11)
    k32 = torch.randint(0, 256, (n, 32), generator=g, device="cuda", dtype=torch.uint8)
    t = timed(lambda: hybrid.x25519_keygen(k32), steps=3)
    pub = hybrid.x25519_keygen(k32)
    res["X25519 KeyGen"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
    t = timed(lambda: hybrid.x25519_shared(k32, pub), steps=3)
    res["X25519 Shared"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
    # the same KeyGen through the C ABI into a preallocated buffer, as the Ed25519 lines below are timed
    t = timed(lambda: check(L.cb200_x25519(k32.data_ptr(), None, pub.data_ptr(), None, n)), steps=3)
    res["X25519 KeyGen (C ABI, preallocated output)"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
    for mlen in (32, 1024):
        msg = torch.randint(0, 256, (n * mlen + 8,), generator=g, device="cuda", dtype=torch.uint8)
        off = (torch.arange(n + 1, device="cuda", dtype=torch.int64) * mlen).contiguous()
        pk = torch.empty((n, 32), dtype=torch.uint8, device="cuda")
        sk = torch.empty((n, 64), dtype=torch.uint8, device="cuda")
        sig = torch.empty((n, 64), dtype=torch.uint8, device="cuda")
        ok = torch.zeros((n,), dtype=torch.uint8, device="cuda")
        tag = "" if mlen == 32 else " (1 KiB messages)"
        t = timed(lambda: check(L.cb200_ed25519_keygen(k32.data_ptr(), pk.data_ptr(), sk.data_ptr(), n)), steps=3)
        if mlen == 32:
            res["Ed25519 KeyGen"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
        t = timed(lambda: check(L.cb200_ed25519_sign(sk.data_ptr(), 64, msg.data_ptr(), off.data_ptr(), sig.data_ptr(), n)),
                  steps=3)
        res["Ed25519 Sign" + tag] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
        t = timed(lambda: check(L.cb200_ed25519_verify(pk.data_ptr(), 32, msg.data_ptr(), off.data_ptr(), sig.data_ptr(),
                                                       ok.data_ptr(), n)), steps=3)
        res["Ed25519 Verify" + tag] = {"n": n, "ms": t, "per_s": n / (t * 1e-3), "all_valid": bool(ok.all().item())}
    msg = torch.randint(0, 256, (n * 32 + 8,), generator=g, device="cuda", dtype=torch.uint8)
    off = (torch.arange(n + 1, device="cuda", dtype=torch.int64) * 32).contiguous()
    pk = torch.empty((n, 1344), dtype=torch.uint8, device="cuda")
    sk = torch.empty((n, 2560), dtype=torch.uint8, device="cuda")
    sig = torch.empty((n, 2484), dtype=torch.uint8, device="cuda")
    st = torch.zeros((n,), dtype=torch.uint8, device="cuda")
    ok = torch.zeros((n,), dtype=torch.uint8, device="cuda")
    t = timed(lambda: check(L.cb200_eddilithium2_keygen(k32.data_ptr(), pk.data_ptr(), sk.data_ptr(), n)), steps=3)
    res["Ed25519-Dilithium2 KeyGen"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
    t = timed(lambda: check(L.cb200_eddilithium2_sign(sk.data_ptr(), 2560, msg.data_ptr(), off.data_ptr(), sig.data_ptr(),
                                                      st.data_ptr(), n)), steps=2, warm=2)
    res["Ed25519-Dilithium2 Sign"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
    t = timed(lambda: check(L.cb200_eddilithium2_verify(pk.data_ptr(), 1344, msg.data_ptr(), off.data_ptr(), sig.data_ptr(),
                                                        ok.data_ptr(), n)), steps=3)
    res["Ed25519-Dilithium2 Verify"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3), "all_valid": bool(ok.all().item())}
    del msg, off, pk, sk, sig, st, ok, k32, pub
    torch.cuda.empty_cache()


def ed448_lines(res):
    """Ed448 and Ed448-Dilithium3 through the C ABI, device-resident, 2^18 operations, per-op keys, 32-byte and 1 KiB
    messages, empty context, with X448 KeyGen / Shared of the same run for comparison."""
    from circl_b200 import x448
    from circl_b200._ffi import check, lib
    L = lib()
    check(L.cb200_set_stream(torch.cuda.current_stream().cuda_stream))
    n = 1 << 18
    g = torch.Generator(device="cuda").manual_seed(12)
    k56 = torch.randint(0, 256, (n, 56), generator=g, device="cuda", dtype=torch.uint8)
    t = timed(lambda: x448.x448_keygen(k56), steps=3)
    pub = x448.x448_keygen(k56)
    res["X448 KeyGen"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
    t = timed(lambda: x448.x448_shared(k56, pub), steps=3)
    res["X448 Shared"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
    del k56, pub
    k57 = torch.randint(0, 256, (n, 57), generator=g, device="cuda", dtype=torch.uint8)
    for mlen in (32, 1024):
        msg = torch.randint(0, 256, (n * mlen + 8,), generator=g, device="cuda", dtype=torch.uint8)
        off = (torch.arange(n + 1, device="cuda", dtype=torch.int64) * mlen).contiguous()
        pk = torch.empty((n, 57), dtype=torch.uint8, device="cuda")
        sk = torch.empty((n, 114), dtype=torch.uint8, device="cuda")
        sig = torch.empty((n, 114), dtype=torch.uint8, device="cuda")
        ok = torch.zeros((n,), dtype=torch.uint8, device="cuda")
        tag = "" if mlen == 32 else " (1 KiB messages)"
        t = timed(lambda: check(L.cb200_ed448_keygen(k57.data_ptr(), pk.data_ptr(), sk.data_ptr(), n)), steps=3)
        if mlen == 32:
            res["Ed448 KeyGen"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
        t = timed(lambda: check(L.cb200_ed448_sign(sk.data_ptr(), 114, msg.data_ptr(), off.data_ptr(), None, 0,
                                                   sig.data_ptr(), n)), steps=3)
        res["Ed448 Sign" + tag] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
        t = timed(lambda: check(L.cb200_ed448_verify(pk.data_ptr(), 57, msg.data_ptr(), off.data_ptr(), None, 0,
                                                     sig.data_ptr(), ok.data_ptr(), n)), steps=3)
        res["Ed448 Verify" + tag] = {"n": n, "ms": t, "per_s": n / (t * 1e-3), "all_valid": bool(ok.all().item())}
        del msg, off, pk, sk, sig, ok
    msg = torch.randint(0, 256, (n * 32 + 8,), generator=g, device="cuda", dtype=torch.uint8)
    off = (torch.arange(n + 1, device="cuda", dtype=torch.int64) * 32).contiguous()
    pk = torch.empty((n, 2009), dtype=torch.uint8, device="cuda")
    sk = torch.empty((n, 4057), dtype=torch.uint8, device="cuda")
    sig = torch.empty((n, 3407), dtype=torch.uint8, device="cuda")
    st = torch.zeros((n,), dtype=torch.uint8, device="cuda")
    ok = torch.zeros((n,), dtype=torch.uint8, device="cuda")
    t = timed(lambda: check(L.cb200_eddilithium3_keygen(k57.data_ptr(), pk.data_ptr(), sk.data_ptr(), n)), steps=3)
    res["Ed448-Dilithium3 KeyGen"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
    t = timed(lambda: check(L.cb200_eddilithium3_sign(sk.data_ptr(), 4057, msg.data_ptr(), off.data_ptr(), sig.data_ptr(),
                                                      st.data_ptr(), n)), steps=2, warm=2)
    res["Ed448-Dilithium3 Sign"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
    t = timed(lambda: check(L.cb200_eddilithium3_verify(pk.data_ptr(), 2009, msg.data_ptr(), off.data_ptr(), sig.data_ptr(),
                                                        ok.data_ptr(), n)), steps=3)
    res["Ed448-Dilithium3 Verify"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3), "all_valid": bool(ok.all().item())}
    del msg, off, pk, sk, sig, st, ok, k57
    torch.cuda.empty_cache()


def hpke_lines(res):
    """HPKE DHKEM(X25519, HKDF-SHA256) and DHKEM(X448, HKDF-SHA512) through the C ABI, device-resident, 2^18 operations,
    per-op and shared receiver keys, with X25519 / X448 KeyGen and Shared of the same run beside them; the time of the
    KDF kernels alone (profiling class hpke) is read for the per-op Encaps and Decaps lines."""
    import subprocess
    from circl_b200 import hybrid, x448
    from circl_b200._ffi import check, lib
    L = lib()
    check(L.cb200_set_stream(torch.cuda.current_stream().cuda_stream))
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        res["card"] = q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        res["card"] = "unknown"
    n = 1 << 18
    g = torch.Generator(device="cuda").manual_seed(13)
    names = L.cb200_profile_kernel_count()
    hpke_kid = [L.cb200_profile_kernel_name(i).decode() for i in range(names)].index("hpke")

    def kdf_ms(fn):
        """(wall ms, KDF kernel ms) of one call, with per-kernel event timing on."""
        import ctypes as C
        check(L.cb200_profile_enable(1))
        fn()
        torch.cuda.synchronize()
        ms = (C.c_double * names)()
        cnt = (C.c_uint64 * names)()
        check(L.cb200_profile_read(ms, cnt, names))
        check(L.cb200_profile_enable(0))
        return ms[hpke_kid]

    for kid, w, nss, curve in ((0x20, 32, 32, "X25519"), (0x21, 56, 64, "X448")):
        name = "DHKEM(X25519, HKDF-SHA256)" if kid == 0x20 else "DHKEM(X448, HKDF-SHA512)"
        k = torch.randint(0, 256, (n, w), generator=g, device="cuda", dtype=torch.uint8)
        kg, sh = (hybrid.x25519_keygen, hybrid.x25519_shared) if kid == 0x20 else (x448.x448_keygen, x448.x448_shared)
        t = timed(lambda: kg(k), steps=3)
        pub = kg(k)
        res[f"{curve} KeyGen"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
        t = timed(lambda: sh(k, pub), steps=3)
        res[f"{curve} Shared"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
        del pub
        seeds = torch.randint(0, 256, (n, w), generator=g, device="cuda", dtype=torch.uint8)
        pk = torch.empty((n, w), dtype=torch.uint8, device="cuda")
        sk = torch.empty((n, w), dtype=torch.uint8, device="cuda")
        enc = torch.empty((n, w), dtype=torch.uint8, device="cuda")
        ss = torch.empty((n, nss), dtype=torch.uint8, device="cuda")
        ss2 = torch.empty((n, nss), dtype=torch.uint8, device="cuda")
        st = torch.zeros((n,), dtype=torch.uint8, device="cuda")
        P = lambda x: x.data_ptr()  # noqa: E731
        ops = {
            "KeyGen": lambda: check(L.cb200_hpke_keygen(kid, P(seeds), P(pk), P(sk), n)),
            "Encaps": lambda: check(L.cb200_hpke_encaps(kid, P(pk), w, P(k), P(enc), P(ss), P(st), n)),
            "Decaps": lambda: check(L.cb200_hpke_decaps(kid, P(sk), w, P(enc), P(ss2), P(st), n)),
            "Encaps (shared pkR)": lambda: check(L.cb200_hpke_encaps(kid, P(pk), 0, P(k), P(enc), P(ss), P(st), n)),
            "Decaps (shared skR)": lambda: check(L.cb200_hpke_decaps(kid, P(sk), 0, P(enc), P(ss2), P(st), n)),
            "AuthEncaps": lambda: check(L.cb200_hpke_auth_encaps(kid, P(pk), w, P(sk), w, P(k), P(enc), P(ss), P(st), n)),
            "AuthDecaps": lambda: check(L.cb200_hpke_auth_decaps(kid, P(sk), w, P(enc), P(pk), w, P(ss2), P(st), n)),
            "AuthEncaps (shared pkR, skS)": lambda: check(L.cb200_hpke_auth_encaps(kid, P(pk), 0, P(sk), 0, P(k), P(enc),
                                                                                   P(ss), P(st), n)),
            "AuthDecaps (shared skR, pkS)": lambda: check(L.cb200_hpke_auth_decaps(kid, P(sk), 0, P(enc), P(pk), 0,
                                                                                   P(ss2), P(st), n)),
        }
        for op, fn in ops.items():
            t = timed(fn, steps=3)
            line = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
            if op in ("KeyGen", "Encaps", "Decaps"):
                line["kdf_ms"] = kdf_ms(fn)
            if op.startswith("Decaps") or op.startswith("AuthDecaps"):
                torch.cuda.synchronize()
                line["roundtrip_ok"] = bool(torch.equal(ss, ss2)) and st.sum().item() == 0
            res[f"{name} {op}"] = line
        del k, seeds, pk, sk, enc, ss, ss2, st
        torch.cuda.empty_cache()


def frodo_lines(res):
    """FrodoKEM-640-SHAKE through the C ABI, device-resident, 2^16 operations: KeyGen, Encaps and Decaps with per-op
    keys, Encaps with one shared pk and Decaps with one shared sk (the tensor-core path), each with the time of its
    frodo and frodo_gemm kernels (profiling classes) read in a separate profiled call; and the oracle's batch function
    on every host thread over the same 2^16 operations, its outputs compared with the GPU's."""
    import ctypes as C
    import subprocess
    from circl_b200._ffi import check, lib
    from oracle import frodo as O
    L = lib()
    check(L.cb200_set_stream(torch.cuda.current_stream().cuda_stream))
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        res["card"] = q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        res["card"] = "unknown"
    n = 1 << 16
    g = torch.Generator(device="cuda").manual_seed(17)
    names = L.cb200_profile_kernel_count()
    kn = [L.cb200_profile_kernel_name(i).decode() for i in range(names)]
    fk, gk = kn.index("frodo"), kn.index("frodo_gemm")

    def split_ms(fn):
        check(L.cb200_profile_enable(1))
        fn()
        torch.cuda.synchronize()
        ms, cnt = (C.c_double * names)(), (C.c_uint64 * names)()
        check(L.cb200_profile_read(ms, cnt, names))
        check(L.cb200_profile_enable(0))
        return ms[fk], ms[gk]

    seeds = torch.randint(0, 256, (n, 48), generator=g, device="cuda", dtype=torch.uint8)
    es = torch.randint(0, 256, (n, 16), generator=g, device="cuda", dtype=torch.uint8)
    pk = torch.empty((n, 9616), dtype=torch.uint8, device="cuda")
    sk = torch.empty((n, 19888), dtype=torch.uint8, device="cuda")
    ct = torch.empty((n, 9720), dtype=torch.uint8, device="cuda")
    ct0 = torch.empty((n, 9720), dtype=torch.uint8, device="cuda")
    ss, ss2 = (torch.empty((n, 16), dtype=torch.uint8, device="cuda") for _ in range(2))
    ss0, ss02 = (torch.empty((n, 16), dtype=torch.uint8, device="cuda") for _ in range(2))
    P = lambda x: x.data_ptr()  # noqa: E731
    ops = {
        "KeyGen": lambda: check(L.cb200_frodo640shake_keygen(P(seeds), P(pk), P(sk), n)),
        "Encaps": lambda: check(L.cb200_frodo640shake_encaps(P(pk), 9616, P(es), P(ct), P(ss), n)),
        "Decaps": lambda: check(L.cb200_frodo640shake_decaps(P(sk), 19888, P(ct), P(ss2), n)),
        "Encaps (shared pk)": lambda: check(L.cb200_frodo640shake_encaps(P(pk), 0, P(es), P(ct0), P(ss0), n)),
        "Decaps (shared sk)": lambda: check(L.cb200_frodo640shake_decaps(P(sk), 0, P(ct0), P(ss02), n)),
    }
    for op, fn in ops.items():
        t = timed(fn, steps=3)
        f_ms, g_ms = split_ms(fn)
        line = {"n": n, "ms": t, "per_s": n / (t * 1e-3), "frodo_ms": f_ms, "frodo_gemm_ms": g_ms}
        if op.startswith("Decaps"):
            torch.cuda.synchronize()
            line["roundtrip_ok"] = bool(torch.equal(ss, ss2)) if op == "Decaps" else bool(torch.equal(ss0, ss02))
        res[f"FrodoKEM-640-SHAKE {op}"] = line
    threads = os.cpu_count() or 1
    hs, hes, hpk, hsk, hct = (x.cpu().numpy() for x in (seeds, es, pk, sk, ct))
    import time
    for op, fn in (("KeyGen", lambda: O.keygen_batch(hs, threads)), ("Encaps", lambda: O.encaps_batch(hpk, hes, threads)),
                   ("Decaps", lambda: O.decaps_batch(hsk, hct, threads))):
        t0 = time.perf_counter()
        out = fn()
        dt = time.perf_counter() - t0
        res[f"FrodoKEM-640-SHAKE {op} oracle"] = {"n": n, "threads": threads, "ms": dt * 1e3, "per_s": n / dt}
        gpu = (pk, sk) if op == "KeyGen" else (ct, ss) if op == "Encaps" else (ss2,)
        out = out if isinstance(out, tuple) else (out,)
        res[f"FrodoKEM-640-SHAKE {op} oracle"]["matches_gpu"] = all(
            bool(np.array_equal(o, g.cpu().numpy())) for o, g in zip(out, gpu))
    del seeds, es, pk, sk, ct, ct0, ss, ss2, ss0, ss02
    torch.cuda.empty_cache()


def _nist_setup(res):
    """The library on torch's stream, and the card and its power limit into res."""
    import subprocess
    from circl_b200._ffi import check, lib
    L = lib()
    check(L.cb200_set_stream(torch.cuda.current_stream().cuda_stream))
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        res["card"] = q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        res["card"] = "unknown"
    return L


def _split_ms(L, fn, c):
    """(ms of kernel class c, ms of class hpke) of one call of fn, with per-kernel event timing on."""
    import ctypes as C
    from circl_b200._ffi import check
    names = L.cb200_profile_kernel_count()
    kn = [L.cb200_profile_kernel_name(i).decode() for i in range(names)]
    check(L.cb200_profile_enable(1))
    fn()
    torch.cuda.synchronize()
    ms = (C.c_double * names)()
    cnt = (C.c_uint64 * names)()
    check(L.cb200_profile_read(ms, cnt, names))
    check(L.cb200_profile_enable(0))
    return ms[kn.index(c)], ms[kn.index("hpke")]


def p256_lines(res):
    """P-256 raw KeyGen / Shared and DHKEM(P-256, HKDF-SHA256) through the C ABI, device-resident, 2^16 operations, per-op
    and shared keys, with X25519 KeyGen / Shared of the same run beside them; the card and its power limit; and the
    time of the curve kernels (profiling class p256) and of the KDF kernels (class hpke) for every DHKEM line, read in
    a separate profiled call."""
    from circl_b200 import hybrid
    L = _nist_setup(res)
    n = 1 << 16
    g = torch.Generator(device="cuda").manual_seed(17)
    k = torch.randint(0, 256, (n, 32), generator=g, device="cuda", dtype=torch.uint8)
    t = timed(lambda: hybrid.x25519_keygen(k), steps=3)
    res["X25519 KeyGen"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
    pub = hybrid.x25519_keygen(k)
    t = timed(lambda: hybrid.x25519_shared(k, pub), steps=3)
    res["X25519 Shared"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
    del pub, k
    torch.cuda.empty_cache()
    nist_lines(res, L, "p256", 32, 32, "P-256", "DHKEM(P-256, HKDF-SHA256)", n, g)


def nist_lines(res, L, c, B, nss, curve, name, n, g):
    """Raw KeyGen / Shared and every DHKEM line of one NIST curve (entry points cb200_<c> and cb200_hpke_<c>_*, B-byte
    scalars, nss-byte shared secrets), each with the time of its curve kernels (<c>_ms) and KDF kernels (hpke_ms)."""
    from circl_b200._ffi import check
    W = 1 + 2 * B
    P = lambda x: x.data_ptr()  # noqa: E731
    H = lambda op: getattr(L, f"cb200_hpke_{c}_{op}")  # noqa: E731
    seeds = torch.randint(0, 256, (n, B), generator=g, device="cuda", dtype=torch.uint8)
    es = torch.randint(0, 256, (n, B), generator=g, device="cuda", dtype=torch.uint8)
    pk = torch.empty((n, W), dtype=torch.uint8, device="cuda")
    sk = torch.empty((n, B), dtype=torch.uint8, device="cuda")
    enc = torch.empty((n, W), dtype=torch.uint8, device="cuda")
    ss = torch.empty((n, nss), dtype=torch.uint8, device="cuda")
    ss2 = torch.empty((n, nss), dtype=torch.uint8, device="cuda")
    st = torch.zeros((n,), dtype=torch.uint8, device="cuda")
    check(H("keygen")(P(seeds), P(pk), P(sk), n))  # valid scalars and points for the raw lines
    raw = torch.empty((n, W), dtype=torch.uint8, device="cuda")
    ecdh = getattr(L, f"cb200_{c}")
    ops = {
        f"{curve} KeyGen": lambda: check(ecdh(P(sk), None, P(raw), P(st), n)),
        f"{curve} Shared": lambda: check(ecdh(P(sk), P(pk), P(raw), P(st), n)),
        f"{name} KeyGen": lambda: check(H("keygen")(P(seeds), P(pk), P(sk), n)),
        f"{name} Encaps": lambda: check(H("encaps")(P(pk), W, P(es), P(enc), P(ss), P(st), n)),
        f"{name} Decaps": lambda: check(H("decaps")(P(sk), B, P(enc), P(ss2), P(st), n)),
        f"{name} Encaps (shared pkR)": lambda: check(H("encaps")(P(pk), 0, P(es), P(enc), P(ss), P(st), n)),
        f"{name} Decaps (shared skR)": lambda: check(H("decaps")(P(sk), 0, P(enc), P(ss2), P(st), n)),
        f"{name} AuthEncaps": lambda: check(H("auth_encaps")(P(pk), W, P(sk), B, P(es), P(enc), P(ss), P(st), n)),
        f"{name} AuthDecaps": lambda: check(H("auth_decaps")(P(sk), B, P(enc), P(pk), W, P(ss2), P(st), n)),
        f"{name} AuthEncaps (shared pkR, skS)": lambda: check(H("auth_encaps")(P(pk), 0, P(sk), 0, P(es), P(enc), P(ss),
                                                                                 P(st), n)),
        f"{name} AuthDecaps (shared skR, pkS)": lambda: check(H("auth_decaps")(P(sk), 0, P(enc), P(pk), 0, P(ss2), P(st),
                                                                                 n)),
    }
    for op, fn in ops.items():
        t = timed(fn, steps=3)
        line = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
        line[f"{c}_ms"], line["hpke_ms"] = _split_ms(L, fn, c)
        if "Decaps" in op:
            torch.cuda.synchronize()
            line["roundtrip_ok"] = bool(torch.equal(ss, ss2)) and st.sum().item() == 0
        res[op] = line
    del seeds, es, pk, sk, enc, ss, ss2, st, raw
    torch.cuda.empty_cache()


def nist_extra_lines(res):
    """The lines of nist_lines for P-384 and P-521 (2^14 operations each), with the card and its power limit."""
    L = _nist_setup(res)
    g = torch.Generator(device="cuda").manual_seed(19)
    n = 1 << 14
    nist_lines(res, L, "p384", 48, 48, "P-384", "DHKEM(P-384, HKDF-SHA384)", n, g)
    nist_lines(res, L, "p521", 66, 64, "P-521", "DHKEM(P-521, HKDF-SHA512)", n, g)


if "--p256" in sys.argv:  # only the P-256 lines above and the X25519 lines they are compared with
    p256_lines(res)
    print(json.dumps(res, indent=1))
    sys.exit(0)


if "--nistp" in sys.argv:  # only the P-384 and P-521 lines
    nist_extra_lines(res)
    print(json.dumps(res, indent=1))
    sys.exit(0)


if "--frodo" in sys.argv:  # only the FrodoKEM lines above
    frodo_lines(res)
    print(json.dumps(res, indent=1))
    sys.exit(0)


if "--hpke" in sys.argv:  # only the HPKE lines above and the curve lines they are compared with
    hpke_lines(res)
    print(json.dumps(res, indent=1))
    sys.exit(0)


if "--ed448" in sys.argv:  # only the Ed448 lines above and the X448 lines they are compared with
    ed448_lines(res)
    print(json.dumps(res, indent=1))
    sys.exit(0)


if "--eddsa" in sys.argv:  # only the signature lines above and the X25519 lines they are compared with
    eddsa_lines(res)
    print(json.dumps(res, indent=1))
    sys.exit(0)


for name, k, log2 in (("ML-KEM-768", 3, 20), ("ML-KEM-1024", 4, 20)):
    scheme = mlkem.ByName(name)
    n = 1 << log2
    g = torch.Generator(device="cuda").manual_seed(1)
    seeds = torch.randint(0, 256, (n, 64), generator=g, device="cuda", dtype=torch.uint8)
    ms = torch.randint(0, 256, (n, 32), generator=g, device="cuda", dtype=torch.uint8)
    t = timed(lambda: scheme.DeriveKeyPairBatch(seeds), steps=3)
    ek, dk = scheme.DeriveKeyPairBatch(seeds)
    res[f"{name} keygen"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
    ct = torch.empty((n, scheme.CiphertextSize()), dtype=torch.uint8, device="cuda")
    ss = torch.empty((n, 32), dtype=torch.uint8, device="cuda")
    t = timed(lambda: scheme.EncapsulateBatch(ek, ms, ct=ct, ss=ss))
    res[f"{name} encaps (per-op ek)"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
    pk0 = scheme.UnmarshalBinaryPublicKey(ek[0].cpu().numpy().tobytes())
    t = timed(lambda: scheme.EncapsulateBatch(pk0, ms, ct=ct, ss=ss))
    res[f"{name} encaps (shared ek)"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
    scheme.EncapsulateBatch(ek, ms, ct=ct, ss=ss)
    ss2 = torch.empty_like(ss)
    t = timed(lambda: scheme.DecapsulateBatch(dk, ct, ss=ss2), steps=3)
    res[f"{name} decaps"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3), "roundtrip_ok": bool(torch.equal(ss, ss2))}
    del seeds, ms, ek, dk, ct, ss, ss2
    torch.cuda.empty_cache()

n = 1 << 19
e = torch.randint(0, 8380417, (n, 256), device="cuda", dtype=torch.int32)
for label, fn in (("Dilithium NTT", lambda: dl.ntt_(e)), ("Dilithium InvNTT", lambda: dl.inv_ntt_(e))):
    t = timed(fn, steps=10)
    res[label] = {"n": n, "ms": t, "per_s": n / (t * 1e-3), "GBps": n * 2048 / (t * 1e-3) / 1e9}
del e
torch.cuda.empty_cache()

# wire-side callers (SURVEY.md 8(f) row 4): X25519, X-Wing, X25519MLKEM768, round-3 Kyber768, all device-resident
from circl_b200 import hybrid  # noqa: E402
n = 1 << 18
g = torch.Generator(device="cuda").manual_seed(2)
k32 = torch.randint(0, 256, (n, 32), generator=g, device="cuda", dtype=torch.uint8)
t = timed(lambda: hybrid.x25519_keygen(k32), steps=3)
pub = hybrid.x25519_keygen(k32)
res["X25519 KeyGen"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
t = timed(lambda: hybrid.x25519_shared(k32, pub), steps=3)
res["X25519 Shared"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
for name in ("X-Wing", "X25519MLKEM768"):
    sch = hybrid.ByName(name)
    seeds = torch.randint(0, 256, (n, sch.SeedSize()), generator=g, device="cuda", dtype=torch.uint8)
    es = torch.randint(0, 256, (n, sch.EncapsulationSeedSize()), generator=g, device="cuda", dtype=torch.uint8)
    t = timed(lambda: sch.DeriveKeyPairBatch(seeds), steps=3)
    pk, sk = sch.DeriveKeyPairBatch(seeds)
    res[f"{name} keygen"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
    t = timed(lambda: sch.EncapsulateBatch(pk, es), steps=3)
    ct, ss = sch.EncapsulateBatch(pk, es)
    res[f"{name} encaps"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
    t = timed(lambda: sch.DecapsulateBatch(sk, ct), steps=3)
    res[f"{name} decaps"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3),
                             "roundtrip_ok": bool(torch.equal(ss, sch.DecapsulateBatch(sk, ct)))}
    del seeds, es, pk, sk, ct, ss
    torch.cuda.empty_cache()
# X448 and the X448 hybrids, device-resident at 2^18
from circl_b200 import x448  # noqa: E402
k56 = torch.randint(0, 256, (n, 56), generator=g, device="cuda", dtype=torch.uint8)
t = timed(lambda: x448.x448_keygen(k56), steps=3)
pub = x448.x448_keygen(k56)
res["X448 KeyGen"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
t = timed(lambda: x448.x448_shared(k56, pub), steps=3)
res["X448 Shared"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
del k56, pub
for sch in x448.All():
    name = sch.Name()
    seeds = torch.randint(0, 256, (n, sch.SeedSize()), generator=g, device="cuda", dtype=torch.uint8)
    es = torch.randint(0, 256, (n, sch.EncapsulationSeedSize()), generator=g, device="cuda", dtype=torch.uint8)
    t = timed(lambda: sch.DeriveKeyPairBatch(seeds), steps=3)
    pk, sk = sch.DeriveKeyPairBatch(seeds)
    res[f"{name} keygen"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
    t = timed(lambda: sch.EncapsulateBatch(pk, es), steps=3)
    ct, ss = sch.EncapsulateBatch(pk, es)
    res[f"{name} encaps"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
    t = timed(lambda: sch.DecapsulateBatch(sk, ct), steps=3)
    res[f"{name} decaps"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3),
                             "roundtrip_ok": bool(torch.equal(ss, sch.DecapsulateBatch(sk, ct)))}
    del seeds, es, pk, sk, ct, ss
    torch.cuda.empty_cache()
k768 = mlkem.ByName("Kyber768")
seeds = torch.randint(0, 256, (n, 64), generator=g, device="cuda", dtype=torch.uint8)
ms = torch.randint(0, 256, (n, 32), generator=g, device="cuda", dtype=torch.uint8)
ek, dk = k768.DeriveKeyPairBatch(seeds)
t = timed(lambda: k768.EncapsulateBatch(ek, ms), steps=3)
res["Kyber768 (round 3) encaps"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
del seeds, ms, ek, dk
torch.cuda.empty_cache()

# ML-DSA family, device-resident through the C ABI (CUDA events): key generation, signing and verification for
# ML-DSA-44/65/87 and round-3 Dilithium3 (SURVEY.md 8(f) rows 2-4); per-op keys, 32-byte messages
from circl_b200 import mldsa  # noqa: E402
from circl_b200._ffi import check, lib  # noqa: E402

L = lib()
n = 1 << 17
g = torch.Generator(device="cuda").manual_seed(9)
dseeds = torch.randint(0, 256, (n, 32), generator=g, device="cuda", dtype=torch.uint8)
msg_d = torch.randint(0, 256, (n * 32 + 8,), generator=g, device="cuda", dtype=torch.uint8)
off_d = (torch.arange(n + 1, device="cuda", dtype=torch.int64) * 32).contiguous()
check(L.cb200_set_stream(torch.cuda.current_stream().cuda_stream))
for name, mode in (("ML-DSA-44", 44), ("ML-DSA-65", 65), ("ML-DSA-87", 87), ("Dilithium3", 3)):
    sch = mldsa.ByName(name)
    pk = torch.empty((n, sch.PublicKeySize()), dtype=torch.uint8, device="cuda")
    sk = torch.empty((n, sch.PrivateKeySize()), dtype=torch.uint8, device="cuda")
    sig = torch.empty((n, sch.SignatureSize()), dtype=torch.uint8, device="cuda")
    st = torch.zeros((n,), dtype=torch.uint8, device="cuda")
    ok = torch.zeros((n,), dtype=torch.uint8, device="cuda")
    t = timed(lambda: check(L.cb200_mldsa_keygen(mode, dseeds.data_ptr(), pk.data_ptr(), sk.data_ptr(), n)), steps=3)
    res[f"{name} keygen"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
    t = timed(lambda: check(L.cb200_mldsa_sign(mode, sk.data_ptr(), sch.PrivateKeySize(), msg_d.data_ptr(), off_d.data_ptr(),
                                               None, 0, None, sig.data_ptr(), st.data_ptr(), n, 0, None)), steps=2, warm=2)
    res[f"{name} sign"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3)}
    t = timed(lambda: check(L.cb200_mldsa_verify(mode, pk.data_ptr(), sch.PublicKeySize(), msg_d.data_ptr(), off_d.data_ptr(),
                                                 None, 0, sig.data_ptr(), ok.data_ptr(), n, 0)), steps=3)
    res[f"{name} verify"] = {"n": n, "ms": t, "per_s": n / (t * 1e-3), "all_valid": bool(ok.all().item())}
    del pk, sk, sig
    torch.cuda.empty_cache()
eddsa_lines(res)
print(json.dumps(res, indent=1))
