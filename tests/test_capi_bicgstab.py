"""CPU tier: the solver entry points b200_invert_bicgstab and b200_invert_cg refuse null arguments, and without a GPU refuse a
real call the way every compute entry point does (no CPU fallback); their Python wrappers refuse a wrong-precision x or b."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest

from quda_b200 import dirac as DR
from quda_b200 import lib as L


def _dirac(lib, buf):
    """a Wilson-PC operator over host memory: creating one only records descriptors, it touches no device"""
    h = C.c_void_p()
    X = (C.c_int * 4)(4, 4, 4, 4)
    g = L.Gauge(buf.ctypes.data, 0, 1, 18, 1.0, 1.0, -1, 1, 1)
    assert lib.b200_dirac_create(C.byref(h), L.DIRAC_WILSONPC, 8, X, C.byref(g), None, None, 0.12, 0, None, None) == 0
    return h


def _refuses_null_arguments(entry):
    lib = L.load()
    solve = getattr(lib, entry)
    buf = np.zeros(1 << 16, dtype=np.uint8)
    sp = L.Spinor(buf.ctypes.data, None, 0, 128, 1)
    p = L.SolverParam()
    assert solve(None, None, C.byref(sp), C.byref(sp), C.byref(p)) == -1  # B200_ERR_INVALID
    assert b"null argument" in lib.b200_last_error()
    h = _dirac(lib, buf)
    try:
        assert solve(h, None, C.byref(sp), C.byref(sp), None) == -1
        assert b"null argument" in lib.b200_last_error()
    finally:
        lib.b200_dirac_destroy(h)


def _refuses_without_a_gpu(entry):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    lib = L.load()
    solve = getattr(lib, entry)
    buf = np.zeros(1 << 16, dtype=np.uint8)
    sp = L.Spinor(buf.ctypes.data, None, 0, 128, 1)
    p = L.SolverParam()
    p.tol, p.maxiter = 1e-10, 10
    h = _dirac(lib, buf)
    try:
        assert solve(h, None, C.byref(sp), C.byref(sp), C.byref(p)) == -4  # B200_ERR_NO_DEVICE
        assert b"no CPU path" in lib.b200_last_error()
    finally:
        lib.b200_dirac_destroy(h)


def test_bicgstab_refuses_null_arguments():
    _refuses_null_arguments("b200_invert_bicgstab")


def test_bicgstab_refuses_without_a_gpu():
    _refuses_without_a_gpu("b200_invert_bicgstab")


def test_cg_refuses_null_arguments():
    _refuses_null_arguments("b200_invert_cg")


def test_cg_refuses_without_a_gpu():
    _refuses_without_a_gpu("b200_invert_cg")


@pytest.mark.parametrize("invert", [DR.invert_cg, DR.invert_bicgstab], ids=["cg", "bicgstab"])
def test_solver_wrappers_refuse_a_precision_mismatch(invert):
    """the C ABI reads x and b in the precise operator's precision, so the wrapper must refuse anything else before the
    call (the stand-ins have no library handle: reaching the call would fail differently)"""
    precise = SimpleNamespace(prec=8)
    for x, b in ((SimpleNamespace(prec=4), SimpleNamespace(prec=8)), (SimpleNamespace(prec=8), SimpleNamespace(prec=4))):
        with pytest.raises(L.B200Error, match="precision"):
            invert(precise, None, x, b)
