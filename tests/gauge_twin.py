"""The test-only host twin of the gauge force, link update, momentum action and plaquette (tests/gaugetwin): the library's
entry points and site code compiled for the CPU.  B200_GAUGE_TWIN_LIB selects another build of it (the sanitizer run)."""
import ctypes as C
import os
import subprocess

from quda_b200 import lib as L

DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "gaugetwin")
_twin = None


def gauge_twin():
    """the CDLL with twin_gauge_force / twin_update_gauge / twin_mom_action / twin_plaquette / twin_last_error declared"""
    global _twin
    if _twin is None:
        path = os.environ.get("B200_GAUGE_TWIN_LIB")
        if not path:
            subprocess.check_call(["make", "-s", "-C", DIR])
            path = os.path.join(DIR, "_build", "libgaugetwin.so")
        _twin = L.declare_gauge(C.CDLL(path), "twin")
    return _twin
