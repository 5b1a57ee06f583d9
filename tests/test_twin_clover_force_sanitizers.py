"""CPU tier: the clover force twin (tests/forcetwin) rebuilt with AddressSanitizer + UndefinedBehaviorSanitizer runs the twin cases of the clover
force in a subprocess (LD_PRELOAD=libasan).  The twin executes the kernels' site code and index maps, so an out-of-bounds
access found here is one the CUDA kernels would commit."""
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
TWIN = os.path.join(HERE, "forcetwin")


def test_clover_force_twin_is_clean_under_asan_and_ubsan():
    p = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not (os.path.isabs(p) and os.path.exists(p)):
        pytest.skip("no libasan in this toolchain")
    subprocess.check_call(["make", "-s", "-C", TWIN, "asan"])  # ~10 s
    env = dict(os.environ, LD_PRELOAD=p, ASAN_OPTIONS="detect_leaks=0", UBSAN_OPTIONS="print_stacktrace=1:halt_on_error=1",
               B200_FORCE_TWIN_LIB=os.path.join(TWIN, "_build", "libforcetwin_asan.so"), OMP_NUM_THREADS="4")
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-s", "-p", "no:cacheprovider",
                        os.path.join(HERE, "test_twin_clover_force.py"), "-k", "twin_matches or deterministic or refuses"],
                       capture_output=True, text=True, env=env, timeout=1500)
    tail = (r.stdout + r.stderr)[-4000:]
    assert "AddressSanitizer" not in r.stdout + r.stderr and "runtime error" not in r.stdout + r.stderr, tail
    assert r.returncode == 0 and " passed" in r.stdout, tail
