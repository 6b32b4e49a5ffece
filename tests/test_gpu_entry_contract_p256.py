"""The argument contract of the P-256 entry points (cb200_p256 and cb200_hpke_p256_*), in the four cases of
tests/test_gpu_entry_contract.py: n = 0; n = 0 with a required pointer null; one host buffer among device buffers;
and device pointers at an odd byte, which these entry points accept (their 65-byte rows are read byte by byte)."""
import pytest

from test_gpu_entry_contract import CUR, ERR_ARG, E, N, _call, env  # noqa: F401  (env is the shared fixture)

pytestmark = pytest.mark.gpu

TABLE = [
    E("cb200_p256", ["s", None, "pk", "st", N], "s", CUR, "s", label="p256_keygen"),
    E("cb200_p256", ["s", "pk", "ss", "st", N], "ss", CUR, "pk", label="p256_shared"),
    E("cb200_hpke_p256_keygen", ["s", "pk", "sk", N], "sk", CUR, "s"),
    E("cb200_hpke_p256_encaps", ["pk", 65, "s", "ct", "ss", "st", N], "pk", CUR, "ss"),
    E("cb200_hpke_p256_decaps", ["sk", 32, "ct", "ss", "st", N], "ct", CUR, "sk"),
    E("cb200_hpke_p256_auth_encaps", ["pk", 65, "sk", 32, "s", "ct", "ss", "st", N], "sk", CUR, "s"),
    E("cb200_hpke_p256_auth_decaps", ["sk", 32, "ct", "pk", 65, "ss", "st", N], "pk", CUR, "st"),
]
ROWS = ["s", "pk", "sk", "ct", "ss"]


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
    # any byte: the all-zero keys are invalid, which a device-pointer call reports through status only
    for a in ROWS:
        if a in e.args:
            rc, err = _call(L, e, ptrs, hostp, 1, shift=a)
            assert rc == 0, (a, rc, err)


def test_status_required_on_device(env):  # noqa: F811
    L, ptrs, host = env
    for e in TABLE[3:]:
        args = [None if a == "st" else a for a in e.args]
        rc, err = _call(L, E(e.fn, args, e.null, e.null_rc), ptrs, host.ctypes.data, 1)
        assert rc == ERR_ARG and "status" in err, (e.fn, rc, err)
