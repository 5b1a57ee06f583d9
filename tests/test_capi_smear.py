"""C ABI of gauge smearing: the entry point is exported, and without a GPU it returns B200_ERR_NO_DEVICE once its
arguments are valid (the library has no CPU path)."""
import ctypes as C

import numpy as np
import pytest

from quda_b200 import lib as L


def test_symbol_exported():
    lib = L.load()
    assert hasattr(lib, "b200_gauge_smear") and "b200_gauge_smear" in L.EXPORTED_SYMBOLS


def test_entry_point_needs_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    lib = L.load()
    buf = np.zeros(64)
    p = buf.ctypes.data
    q = (C.c_void_p * 4)(p, p, p, p)
    X = (C.c_int * 4)(4, 4, 4, 4)
    c = (C.c_double * 3)(0.75, 0.6, 0.3)
    for type_ in (L.SMEAR_APE, L.SMEAR_STOUT, L.SMEAR_OVRIMP_STOUT, L.SMEAR_HYP):
        assert lib.b200_gauge_smear(q, q, X, 8, type_, c, -1, 2, None) == -4  # B200_ERR_NO_DEVICE
    # invalid arguments are refused before the device is looked for
    assert lib.b200_gauge_smear(q, q, X, 8, 4, c, -1, 2, None) == -1
    assert lib.b200_gauge_smear(q, q, X, 8, L.SMEAR_HYP, c, -1, 0, None) == -1
