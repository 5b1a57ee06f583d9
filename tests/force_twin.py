"""The test-only host twin of the clover force (tests/forcetwin): the library's b200_clover_force_accumulate entry point and
site code compiled for the CPU.  B200_FORCE_TWIN_LIB selects another build of it (the sanitizer run)."""
import ctypes as C
import os
import subprocess

from quda_b200 import lib as L

DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "forcetwin")
_twin = None


def force_twin():
    """the CDLL with twin_clover_force_accumulate / twin_last_error declared"""
    global _twin
    if _twin is None:
        path = os.environ.get("B200_FORCE_TWIN_LIB")
        if not path:
            subprocess.check_call(["make", "-s", "-C", DIR])
            path = os.path.join(DIR, "_build", "libforcetwin.so")
        _twin = L.declare_clover_force(C.CDLL(path), "twin")
    return _twin
