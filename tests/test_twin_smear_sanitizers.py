"""CPU tier: the smearing twin (tests/smeartwin) rebuilt with AddressSanitizer + UndefinedBehaviorSanitizer runs the twin
cases of gauge smearing in a subprocess (LD_PRELOAD=libasan).  The twin executes the kernels' site code, index maps,
decorated-link slots and launch sequence, so an out-of-bounds access found here is one the CUDA kernels would commit."""
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
TWIN = os.path.join(HERE, "smeartwin")


def test_smear_twin_is_clean_under_asan_and_ubsan():
    p = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not (os.path.isabs(p) and os.path.exists(p)):
        pytest.skip("no libasan in this toolchain")
    subprocess.check_call(["make", "-s", "-C", TWIN, "asan"])
    env = dict(os.environ, LD_PRELOAD=p, ASAN_OPTIONS="detect_leaks=0", UBSAN_OPTIONS="print_stacktrace=1:halt_on_error=1",
               B200_SMEAR_TWIN_LIB=os.path.join(TWIN, "_build", "libsmeartwin_asan.so"), OMP_NUM_THREADS="4")
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-s", "-p", "no:cacheprovider",
                        os.path.join(HERE, "test_twin_smear.py"), "-k",
                        "refusals or crafted or compose or zero or (matches_restatement and X1 and near_identity)"],
                       capture_output=True, text=True, env=env, timeout=1500)
    tail = (r.stdout + r.stderr)[-4000:]
    assert "AddressSanitizer" not in r.stdout + r.stderr and "runtime error" not in r.stdout + r.stderr, tail
    assert r.returncode == 0 and " passed" in r.stdout, tail
