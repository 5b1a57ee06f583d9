"""The test-only host twin of the clover construction (tests/clovertwin): the library's b200_compute_clover /
b200_clover_invert_packed entry points and site code compiled for the CPU, as a dslash.Backend."""
import ctypes as C
import os
import subprocess

from quda_b200 import dslash as D
from quda_b200 import lib as L

DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "clovertwin")
_twin = None


def clover_twin():
    global _twin
    if _twin is None:
        subprocess.check_call(["make", "-s", "-C", DIR])
        lib = C.CDLL(os.path.join(DIR, "_build", "libclovertwin.so"))
        L.declare_clover(lib, "twin")
        _twin = D.Backend(lib, "twin")
    return _twin
