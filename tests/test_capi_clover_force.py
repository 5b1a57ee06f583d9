"""C ABI of the clover force: both entry points are exported, and without a GPU each returns B200_ERR_NO_DEVICE once its
arguments are valid (the library has no CPU path)."""
import ctypes as C

import numpy as np
import pytest

from quda_b200 import lib as L


def _no_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    return L.load()


def test_symbols_exported():
    lib = L.load()
    for name in ("b200_clover_force_accumulate", "b200_clover_force"):
        assert hasattr(lib, name) and name in L.EXPORTED_SYMBOLS


def test_accumulate_needs_a_device():
    lib = _no_gpu()
    buf = np.zeros(64)
    p = buf.ctypes.data
    q = (C.c_void_p * 4)(p, p, p, p)
    xs = (C.c_void_p * 2)(p, p)
    rc = lib.b200_clover_force_accumulate(p, q, p, (C.c_int * 4)(4, 4, 4, 4), 8, 2, xs, xs, (C.c_double * 2)(0.1, 0.2),
                                          (C.c_double * 4)(0.1, 0.2, 0.3, 0.4), 0.5, 1, None)
    assert rc == -4  # B200_ERR_NO_DEVICE


def test_operator_level_needs_a_device():
    lib = _no_gpu()
    buf = np.zeros(64)
    p = buf.ctypes.data
    X = (C.c_int * 4)(4, 4, 4, 4)
    g = L.Gauge(p, 0, 1, 18, 1.0, 1.0, 1, 1, 1)
    a = L.Clover(p, 0, 0, 1, 0.0, 1.0)
    h = C.c_void_p()
    assert lib.b200_dirac_create(C.byref(h), L.DIRAC_CLOVERPC, 8, X, C.byref(g), C.byref(a), None, 0.12, 2, None, None) == 0
    try:
        s = (L.Spinor * 1)(L.Spinor(p, None, 0, 128, 1))
        q = (C.c_void_p * 4)(p, p, p, p)
        rc = lib.b200_clover_force(p, 0.1, s, (C.c_double * 1)(1.0), -0.0144, -0.02, 1, 1.0, q, p, h)
        assert rc == -4  # B200_ERR_NO_DEVICE
    finally:
        lib.b200_dirac_destroy(h)
