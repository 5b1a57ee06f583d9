"""C ABI of the gauge force, link update, momentum action and plaquette: the entry points are exported, and without a GPU
each returns B200_ERR_NO_DEVICE once its arguments are valid (the library has no CPU path)."""
import ctypes as C

import numpy as np
import pytest

from quda_b200 import lib as L

NAMES = ("b200_gauge_force", "b200_update_gauge", "b200_mom_action", "b200_plaquette")


def _no_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    return L.load()


def test_symbols_exported():
    lib = L.load()
    for name in NAMES:
        assert hasattr(lib, name) and name in L.EXPORTED_SYMBOLS


def test_entry_points_need_a_device():
    lib = _no_gpu()
    buf = np.zeros(64)
    p = buf.ctypes.data
    q = (C.c_void_p * 4)(p, p, p, p)
    X = (C.c_int * 4)(4, 4, 4, 4)
    paths = np.array([[[(mu + 1) % 4, 7 - mu, 7 - (mu + 1) % 4]] for mu in range(4)], dtype=np.int32)
    rc = lib.b200_gauge_force(p, q, X, 8, paths.ctypes.data_as(C.POINTER(C.c_int)), (C.c_int * 1)(3), (C.c_double * 1)(1.0),
                              1, 3, 0.1, None)
    assert rc == -4  # B200_ERR_NO_DEVICE
    assert lib.b200_update_gauge(q, q, p, X, 8, 0.1, 0, 1, None) == -4
    S = C.c_double()
    assert lib.b200_mom_action(C.byref(S), p, X, 4, None) == -4
    assert lib.b200_plaquette((C.c_double * 3)(), q, X, 8, None) == -4
