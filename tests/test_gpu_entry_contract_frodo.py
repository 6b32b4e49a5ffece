"""The argument contract of the FrodoKEM-640-SHAKE entry points, in the four cases of tests/test_gpu_entry_contract.py
(n = 0, n = 0 with a required pointer null, one host buffer among device buffers, each misaligned device pointer).
Device pointers need 8-byte alignment, so a ciphertext row at an 8-aligned address that is not 16-aligned is accepted:
one Encaps and one Decaps run there on the zero-filled buffers, which are large enough for one operation."""
import pytest

from test_gpu_entry_contract import CUR, ERR_ARG, E, N, _call, env  # noqa: F401  (env is the shared fixture)

pytestmark = pytest.mark.gpu

TABLE = [
    E("cb200_frodo640shake_keygen", ["s", "pk", "sk", N], "sk", CUR, "s", ["s", "pk", "sk"]),
    E("cb200_frodo640shake_encaps", ["pk", 9616, "s", "ct", "ss", N], "pk", CUR, "ss", ["pk", "s", "ct", "ss"]),
    E("cb200_frodo640shake_decaps", ["sk", 19888, "ct", "ss", N], "ct", CUR, "sk", ["sk", "ct", "ss"]),
]


@pytest.mark.parametrize("e", TABLE, ids=[e.id for e in TABLE])
def test_entry_contract(env, e):  # noqa: F811
    L, ptrs, host = env
    hostp = host.ctypes.data
    assert _call(L, e, ptrs, hostp, 0)[0] == 0
    rc, err = _call(L, e, ptrs, hostp, 0, null=e.null)
    assert rc == e.null_rc, err
    if rc:
        assert err.startswith(e.fn + ":"), err
    rc, err = _call(L, e, ptrs, hostp, 1, host=e.mix)
    assert rc == ERR_ARG and err.startswith(e.prefix + ": mixed host/device pointers"), (rc, err)
    for a in e.align:
        rc, err = _call(L, e, ptrs, hostp, 1, shift=a)
        assert rc == ERR_ARG and err.startswith(e.prefix + ":") and "aligned" in err, (a, rc, err)


def test_eight_aligned_ciphertext_is_accepted(env):  # noqa: F811
    """ct at an address that is 8- but not 16-byte aligned runs (the buffers are zero-filled and hold one operation)."""
    import torch
    L, ptrs, _ = env
    assert L.cb200_frodo640shake_encaps(ptrs["pk"], 0, ptrs["s"], ptrs["ct"] + 8, ptrs["ss"], 1) == 0
    assert L.cb200_frodo640shake_decaps(ptrs["sk"], 0, ptrs["ct"] + 8, ptrs["ss"], 1) == 0
    torch.cuda.synchronize()
