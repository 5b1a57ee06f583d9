"""The test-only host twin of the gradient flow and the gauge observables (tests/flowtwin), which also carries the gauge
twin's entry points: the library's entry points and site code compiled for the CPU.  B200_FLOW_TWIN_LIB selects another
build of it (the sanitizer run)."""
import ctypes as C
import os
import subprocess

from quda_b200 import lib as L

DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "flowtwin")
_twin = None


def flow_twin():
    """the CDLL with twin_gauge_flow / twin_gauge_observables, the gauge twin's entry points and twin_last_error declared"""
    global _twin
    if _twin is None:
        path = os.environ.get("B200_FLOW_TWIN_LIB")
        if not path:
            subprocess.check_call(["make", "-s", "-C", DIR])
            path = os.path.join(DIR, "_build", "libflowtwin.so")
        _twin = L.declare_flow(L.declare_gauge(C.CDLL(path), "twin"), "twin")
    return _twin
