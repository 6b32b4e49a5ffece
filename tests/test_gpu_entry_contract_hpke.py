"""The argument contract of the HPKE DHKEM entry points, in the four cases of tests/test_gpu_entry_contract.py (n = 0,
n = 0 with a required pointer null, one host buffer among device buffers, each misaligned device pointer), for both
ids; and an unknown id, which is CB200_ERR_ARG."""
import pytest

from test_gpu_entry_contract import CUR, ERR_ARG, E, N, _call, env  # noqa: F401  (env is the shared fixture)

pytestmark = pytest.mark.gpu

TABLE = []
for kid, w in ((0x20, 32), (0x21, 56)):
    t = "x25519" if kid == 0x20 else "x448"
    TABLE += [
        E("cb200_hpke_keygen", [kid, "s", "pk", "sk", N], "sk", CUR, "s", ["s", "pk", "sk"], label=f"hpke_keygen_{t}"),
        E("cb200_hpke_encaps", [kid, "pk", w, "s", "ct", "ss", "st", N], "pk", CUR, "ss", ["pk", "s", "ct", "ss"],
          label=f"hpke_encaps_{t}"),
        E("cb200_hpke_decaps", [kid, "sk", w, "ct", "ss", "st", N], "ct", CUR, "sk", ["sk", "ct", "ss"],
          label=f"hpke_decaps_{t}"),
        E("cb200_hpke_auth_encaps", [kid, "pk", w, "sk", w, "s", "ct", "ss", "st", N], "sk", CUR, "s",
          ["pk", "sk", "s", "ct", "ss"], label=f"hpke_auth_encaps_{t}"),
        E("cb200_hpke_auth_decaps", [kid, "sk", w, "ct", "pk", w, "ss", "st", N], "pk", CUR, "st",
          ["sk", "ct", "pk", "ss"], label=f"hpke_auth_decaps_{t}"),
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


@pytest.mark.parametrize("e", TABLE[:5], ids=[e.fn for e in TABLE[:5]])
def test_unknown_id(env, e):  # noqa: F811
    L, ptrs, host = env
    for bad in (0x10, 0x22, 0):
        args = [bad] + e.args[1:]
        rc, err = _call(L, E(e.fn, args, e.null, e.null_rc), ptrs, host.ctypes.data, 1)
        assert rc == ERR_ARG and err.startswith(e.fn + ":"), (bad, rc, err)
