"""C ABI of the gradient flow and the gauge observables: the entry points are exported, and without a GPU each returns
B200_ERR_NO_DEVICE once its arguments are valid (the library has no CPU path)."""
import ctypes as C

import numpy as np
import pytest

from quda_b200 import gauge as GP
from quda_b200 import lib as L

NAMES = ("b200_gauge_flow", "b200_gauge_observables")


def test_symbols_exported():
    lib = L.load()
    for name in NAMES:
        assert hasattr(lib, name) and name in L.EXPORTED_SYMBOLS


def test_entry_points_need_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    lib = L.load()
    buf = np.zeros(64)
    p = buf.ctypes.data
    q = (C.c_void_p * 4)(p, p, p, p)
    X = (C.c_int * 4)(4, 4, 4, 4)
    table, lengths, n, ml = GP.path_table(GP.FLOW_ACTIONS["symanzik"][0])
    coeffs = GP.FLOW_ACTIONS["symanzik"][1]
    rc = lib.b200_gauge_flow(q, q, X, 8, table.ctypes.data_as(C.POINTER(C.c_int)), (C.c_int * n)(*lengths),
                             (C.c_double * n)(*coeffs), n, ml, 0.01, 3, None)
    assert rc == -4  # B200_ERR_NO_DEVICE
    assert lib.b200_gauge_observables((C.c_double * 3)(), C.byref(C.c_double()), None, q, X, 4, None) == -4
    # invalid arguments are refused before the device is looked for
    assert lib.b200_gauge_flow(q, q, X, 8, table.ctypes.data_as(C.POINTER(C.c_int)), (C.c_int * n)(*lengths),
                               (C.c_double * n)(*coeffs), n, ml, 0.01, 0, None) == -1
