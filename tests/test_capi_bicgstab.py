"""CPU tier: b200_invert_bicgstab refuses null arguments, and without a GPU refuses a real call the way every compute entry
point does (no CPU fallback)."""
import ctypes as C

import numpy as np
import pytest

from quda_b200 import lib as L


def _dirac(lib, buf):
    """a Wilson-PC operator over host memory: creating one only records descriptors, it touches no device"""
    h = C.c_void_p()
    X = (C.c_int * 4)(4, 4, 4, 4)
    g = L.Gauge(buf.ctypes.data, 0, 1, 18, 1.0, 1.0, -1, 1, 1)
    assert lib.b200_dirac_create(C.byref(h), L.DIRAC_WILSONPC, 8, X, C.byref(g), None, None, 0.12, 0, None, None) == 0
    return h


def test_bicgstab_refuses_null_arguments():
    lib = L.load()
    buf = np.zeros(1 << 16, dtype=np.uint8)
    sp = L.Spinor(buf.ctypes.data, None, 0, 128, 1)
    p = L.SolverParam()
    assert lib.b200_invert_bicgstab(None, None, C.byref(sp), C.byref(sp), C.byref(p)) == -1  # B200_ERR_INVALID
    assert b"null argument" in lib.b200_last_error()
    h = _dirac(lib, buf)
    try:
        assert lib.b200_invert_bicgstab(h, None, C.byref(sp), C.byref(sp), None) == -1
        assert b"null argument" in lib.b200_last_error()
    finally:
        lib.b200_dirac_destroy(h)


def test_bicgstab_refuses_without_a_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    lib = L.load()
    buf = np.zeros(1 << 16, dtype=np.uint8)
    sp = L.Spinor(buf.ctypes.data, None, 0, 128, 1)
    p = L.SolverParam()
    p.tol, p.maxiter = 1e-10, 10
    h = _dirac(lib, buf)
    try:
        assert lib.b200_invert_bicgstab(h, None, C.byref(sp), C.byref(sp), C.byref(p)) == -4  # B200_ERR_NO_DEVICE
        assert b"no CPU path" in lib.b200_last_error()
    finally:
        lib.b200_dirac_destroy(h)
