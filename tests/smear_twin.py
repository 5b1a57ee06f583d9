"""The test-only host twin of gauge smearing (tests/smeartwin), which also carries the flow twin's and the gauge twin's
entry points: the library's entry points and site code compiled for the CPU.  B200_SMEAR_TWIN_LIB selects another build of
it (the sanitizer run)."""
import ctypes as C
import os
import subprocess

from quda_b200 import lib as L

DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "smeartwin")
_twin = None


def smear_twin():
    """the CDLL with twin_gauge_smear, twin_su3_project, the flow and gauge twins' entry points and twin_last_error declared"""
    global _twin
    if _twin is None:
        path = os.environ.get("B200_SMEAR_TWIN_LIB")
        if not path:
            subprocess.check_call(["make", "-s", "-C", DIR])
            path = os.path.join(DIR, "_build", "libsmeartwin.so")
        lib = L.declare_smear(L.declare_flow(L.declare_gauge(C.CDLL(path), "twin"), "twin"), "twin")
        lib.twin_su3_project.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        lib.twin_su3_project.restype = C.c_int
        _twin = lib
    return _twin
