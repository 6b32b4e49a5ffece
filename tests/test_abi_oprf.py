"""CPU-only: the OPRF entry points are exported, report the suite sizes, refuse unknown suites and fail loudly without
a device."""
import ctypes as C

import numpy as np
import pytest

import oprf_model as om

IDS = {3: om.P256, 4: om.P384, 5: om.P521}


def test_exports_and_sizes():
    from circl_b200._ffi import lib
    L = C.CDLL(lib()._name)
    for name in ("derive_key", "evaluate", "full_evaluate", "element_size", "scalar_size", "output_size", "proof_size"):
        assert hasattr(L, "cb200_oprf_" + name), name
    L = lib()
    for sid, s in IDS.items():
        assert (L.cb200_oprf_element_size(sid), L.cb200_oprf_scalar_size(sid), L.cb200_oprf_output_size(sid),
                L.cb200_oprf_proof_size(sid)) == (s.Ne, s.Ns, s.Nh, s.proof_size)
    for bad in (0, 1, 2, 6, -1):
        assert L.cb200_oprf_element_size(bad) == 0


def test_python_suites():
    from circl_b200 import oprf
    assert [oprf.GetSuite(i).Identifier() for i in om.SUITES] == list(om.SUITES)
    with pytest.raises(oprf.ErrInvalidSuite):
        oprf.GetSuite("ristretto255-SHA512")


def test_entry_points_without_a_device():
    from circl_b200 import _ffi
    L = _ffi.lib()
    z = np.zeros(4096, np.uint8)
    p = z.ctypes.data
    off = np.zeros(2, np.uint64)
    assert L.cb200_oprf_derive_key(3, 0, p, None, 0, p, p, 1) == -2
    assert L.cb200_oprf_evaluate(4, 1, p, 0, p, 1, p, None, 0, p, p, p, 1) == -2
    assert L.cb200_oprf_full_evaluate(5, 2, p, 0, p, off.ctypes.data, None, 0, p, p, 1) == -2
