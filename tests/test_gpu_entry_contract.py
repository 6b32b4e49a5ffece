"""The argument contract of every batched C entry point, before any kernel runs.

For each entry point the table below fixes the return code (and, for errors, that the text starts with the function's
name) of:
  * n = 0 with valid device pointers;
  * n = 0 with a required pointer null (the lattice entry points return 0 for an empty batch before they look at
    pointers; the curve entry points check pointers first and return CB200_ERR_ARG);
  * one host buffer among device buffers;
  * one device pointer off by one byte, once per pointer that has an alignment rule.
Every case is refused or returns before a launch, so no kernel ever sees these buffers.  They are still sized for one
operation, zero-filled, so that nothing here can fault.
"""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N = object()  # stands for the batch size in an argument list
ERR_ARG = -1
ROW = 1 << 16  # bytes of every test buffer: more than one operation of any entry point needs


class E:
    def __init__(self, fn, args, null, null_rc, mix=None, align=(), prefix=None, label=None):
        self.fn = fn
        self.args = args            # ints, N, None, or buffer names (str)
        self.null = null            # the required buffer set to null in the n = 0 case
        self.null_rc = null_rc
        self.mix = mix              # the buffer passed as a host pointer (None: single-buffer entry point)
        self.align = align          # buffers with a device alignment rule
        self.prefix = prefix or fn  # error texts start with "<prefix>:"
        self.id = label or fn


LAT, CUR = 0, ERR_ARG  # n = 0 with a null pointer: lattice family / curve family

TABLE = [
    E("cb200_kyber_ntt", ["p", N, 0], "p", LAT, align=["p"]),
    E("cb200_kyber_dot", ["o", "a", "b", 2, N], "a", LAT, "a", ["o", "a", "b"]),
    E("cb200_kyber_mulhat", ["o", "a", "b", N], "a", LAT, "b", ["o", "a", "b"], prefix="cb200_kyber_dot"),
    E("cb200_kyber_poly_op", [0, "o", "a", "b", N], "a", LAT, "b", ["o", "a", "b"]),
    E("cb200_dil_ntt", ["p", N, 1], "p", LAT, align=["p"]),
    E("cb200_dil_dot", ["o", "a", "b", 2, N], "b", LAT, "a", ["o", "a", "b"]),
    E("cb200_dil_mulhat", ["o", "a", "b", N], "b", LAT, "a", ["o", "a", "b"], prefix="cb200_dil_dot"),
    E("cb200_dil_poly_op", [1, "o", "a", "b", N], "o", LAT, "b", ["o", "a", "b"]),
    E("cb200_dil_exceeds", ["p", 100, "f", N], "f", LAT, "f", ["p"]),
    E("cb200_dil_power2round", ["a0", "a1", "a", N], "a", LAT, "a1", ["a0", "a1", "a"]),
    E("cb200_dil_pack_le16", ["o", "p", N], "p", LAT, "p", ["o", "p"]),
    E("cb200_keccak_f1600", ["s", N, 0], "s", LAT, align=["s"]),
    E("cb200_sha3", [256, "i", 32, 32, "o", 32, N], "o", LAT, "i"),
    E("cb200_kyber_derive_uniform", ["p", "s", 32, "xy", N], "s", LAT, "s", ["p"]),
    E("cb200_kyber_derive_noise", ["p", 2, "s", 32, "nn", N], "nn", LAT, "nn", ["p"]),
    E("cb200_kyber_pack", ["o", "p", N], "p", LAT, "p", ["o", "p"]),
    E("cb200_kyber_unpack", ["p", "i", N], "i", LAT, "i", ["p", "i"]),
    E("cb200_kyber_compress", ["o", "p", 4, N], "o", LAT, "p", ["o", "p"]),
    E("cb200_kyber_decompress", ["p", "i", 10, N], "p", LAT, "i", ["p", "i"]),
    E("cb200_dil_derive_uniform", ["p", "s", 32, "nn", N], "s", LAT, "s", ["p", "nn"]),
    E("cb200_dil_derive_leq_eta", [65, "p", "s", 64, "nn", N], "p", LAT, "nn", ["p", "nn"]),
    E("cb200_dil_derive_le_gamma1", [44, "p", "s", 64, "nn", N], "nn", LAT, "s", ["p", "nn"]),
    E("cb200_dil_derive_ball", [87, "p", "s", 64, N], "s", LAT, "s", ["p"]),
    E("cb200_mlkem_encaps", [3, "ek", 1184, "s", "ct", "ss", "st", N], "ek", LAT, "s", ["ek", "s", "ct", "ss"]),
    E("cb200_mlkem_encaps_push", [3, "ek", 1184, "s", "ct", "ss", "st", N, None, None], "ek", LAT, "s",
      ["ek", "s", "ct", "ss"], prefix="cb200_mlkem_encaps"),
    E("cb200_mlkem_decaps", [3, "dk", 2400, "ct", "ss", "st", N], "ct", LAT, "ct", ["dk", "ct", "ss"]),
    E("cb200_mlkem_keygen", [3, "s", "ek", "dk", N], "dk", LAT, "s", ["s", "ek", "dk"]),
    E("cb200_kyber_kem_keygen", [2, "s", "ek", "dk", N], "s", LAT, "ek", ["s", "ek", "dk"]),
    E("cb200_kyber_kem_encaps", [4, "ek", 1568, "s", "ct", "ss", N], "ss", LAT, "s", ["ek", "s", "ct", "ss"]),
    E("cb200_kyber_kem_decaps", [3, "dk", 2400, "ct", "ss", N], "dk", LAT, "ct", ["dk", "ct", "ss"]),
    E("cb200_x25519", ["k", "pt", "o", "st", N], "k", CUR, "pt", ["k", "pt", "o"]),
    E("cb200_x448", ["k", "pt", "o", "st", N], "o", CUR, "st", ["k", "pt", "o"]),
    E("cb200_xwing_keygen", ["s", "pk", N], "s", CUR, "s", ["s", "pk"]),
    E("cb200_xwing_encaps", ["pk", 1216, "s", "ct", "ss", "st", N], "pk", CUR, "s", ["pk", "s", "ct", "ss"]),
    E("cb200_xwing_decaps", ["sk", 32, "ct", "ss", N], "ss", CUR, "ct", ["sk", "ct", "ss"]),
    E("cb200_hybrid_keygen", [0, "s", "pk", "sk", N], "s", CUR, "pk", ["s", "pk", "sk"], label="hybrid_keygen_x25519"),
    E("cb200_hybrid_keygen", [3, "s", "pk", "sk", N], "sk", CUR, "s", ["s", "pk", "sk"], label="hybrid_keygen_x448"),
    E("cb200_hybrid_encaps", [1, "pk", 1216, "s", "ct", "ss", "st", N], "pk", CUR, "s", ["pk", "s", "ct", "ss"],
      label="hybrid_encaps_x25519"),
    E("cb200_hybrid_encaps", [4, "pk", 1624, "s", "ct", "ss", "st", N], "ss", CUR, "st", ["pk", "s", "ct", "ss"],
      label="hybrid_encaps_x448"),
    E("cb200_hybrid_decaps", [2, "sk", 1664, "ct", "ss", "st", N], "sk", CUR, "ct", ["sk", "ct", "ss"],
      label="hybrid_decaps_x25519"),
    E("cb200_hybrid_decaps", [3, "sk", 2456, "ct", "ss", "st", N], "ct", CUR, "st", ["sk", "ct", "ss"],
      label="hybrid_decaps_x448"),
    E("cb200_mldsa_sign", [44, "sk", 2560, "m", "mo", None, 0, "r", "sig", "st", N, 0, None], "sk", LAT, "m",
      ["sk", "mo"]),
    E("cb200_mldsa_verify", [87, "pk", 2592, "m", "mo", None, 0, "sig", "ok", N, 0], "ok", LAT, "sig", ["pk", "mo"]),
    E("cb200_mldsa_keygen", [2, "s", "pk", "sk", N], "pk", LAT, "sk", ["s", "pk", "sk"]),
    E("cb200_mldsa65_sign", ["sk", 4032, "m", "mo", None, 0, None, "sig", None, N, 0, None], "sig", LAT, "sk",
      ["sk", "mo"], prefix="cb200_mldsa_sign"),
    E("cb200_mldsa65_verify", ["pk", 1952, "m", "mo", None, 0, "sig", "ok", N, 0], "pk", LAT, "mo", ["pk", "mo"],
      prefix="cb200_mldsa_verify"),
    E("cb200_mldsa65_keygen", ["s", "pk", "sk", N], "s", LAT, "pk", ["s", "pk", "sk"], prefix="cb200_mldsa_keygen"),
    E("cb200_ed25519_keygen", ["s", "pk", "sk", N], "s", CUR, "sk", ["s", "pk", "sk"]),
    E("cb200_ed25519_sign", ["sk", 64, "m", "mo", "sig", N], "m", CUR, "m", ["sk", "mo", "sig"]),
    E("cb200_ed25519_verify", ["pk", 32, "m", "mo", "sig", "ok", N], "ok", CUR, "ok", ["pk", "mo", "sig"]),
    E("cb200_eddilithium2_keygen", ["s", "pk", "sk", N], "sk", CUR, "s", ["s", "pk", "sk"]),
    E("cb200_eddilithium2_sign", ["sk", 2560, "m", "mo", "sig", "st", N], "sig", CUR, "st", ["sk", "mo", "sig"]),
    E("cb200_eddilithium2_verify", ["pk", 1344, "m", "mo", "sig", "ok", N], "mo", CUR, "sig", ["pk", "mo", "sig"]),
    E("cb200_ed448_keygen", ["s", "pk", "sk", N], "pk", CUR, "sk"),
    E("cb200_ed448_sign", ["sk", 114, "m", "mo", None, 0, "sig", N], "sk", CUR, "sig", ["mo"]),
    E("cb200_ed448_verify", ["pk", 57, "m", "mo", None, 0, "sig", "ok", N], "sig", CUR, "m", ["mo"]),
    E("cb200_eddilithium3_keygen", ["s", "pk", "sk", N], "s", CUR, "pk"),
    E("cb200_eddilithium3_sign", ["sk", 4057, "m", "mo", "sig", "st", N], "mo", CUR, "sk", ["mo"]),
    E("cb200_eddilithium3_verify", ["pk", 2009, "m", "mo", "sig", "ok", N], "ok", CUR, "pk", ["mo"]),
]


@pytest.fixture(scope="module")
def env():
    import torch

    import circl_b200
    from circl_b200 import _ffi
    circl_b200.init(0)
    names = sorted({a for e in TABLE for a in e.args if isinstance(a, str)})
    dev = {a: torch.zeros(ROW, dtype=torch.uint8, device="cuda") for a in names}
    host = np.zeros(ROW, dtype=np.uint8)
    torch.cuda.synchronize()
    yield _ffi.lib(), {a: t.data_ptr() for a, t in dev.items()}, host
    torch.cuda.synchronize()
    circl_b200.shutdown()


def _call(L, e, ptrs, hostp, n, null=None, host=None, shift=None):
    argv = []
    for a in e.args:
        if a is N:
            argv.append(n)
        elif isinstance(a, str):
            if a == null:
                argv.append(None)
            elif a == host:
                argv.append(hostp)
            else:
                argv.append(ptrs[a] + (1 if a == shift else 0))
        else:
            argv.append(a)
    rc = getattr(L, e.fn)(*argv)
    return rc, L.cb200_last_error().decode()


@pytest.mark.parametrize("e", TABLE, ids=[e.id for e in TABLE])
def test_entry_contract(env, e):
    L, ptrs, host = env
    hostp = host.ctypes.data
    assert _call(L, e, ptrs, hostp, 0)[0] == 0
    rc, err = _call(L, e, ptrs, hostp, 0, null=e.null)
    assert rc == e.null_rc, err
    if rc:
        assert err.startswith(e.fn + ":"), err
    if e.mix is not None:
        rc, err = _call(L, e, ptrs, hostp, 1, host=e.mix)
        assert rc == ERR_ARG and err.startswith(e.prefix + ": mixed host/device pointers"), (rc, err)
    for a in e.align:
        rc, err = _call(L, e, ptrs, hostp, 1, shift=a)
        assert rc == ERR_ARG and err.startswith(e.prefix + ":") and "aligned" in err, (a, rc, err)
