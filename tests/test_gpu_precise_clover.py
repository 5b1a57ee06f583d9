"""GPU tier of the per-element bounds of tests/precise_clover.py: the clover build and the clover force of
libquda_b200.so on the cases of the CPU tier, in fp64 bit for bit against the host twins and between repeated calls
(the trlog reduction on ragged grids included), the extended-lattice build for every border mask on one GPU, and one
larger build."""
import numpy as np
import pytest

import precise_clover_cases as C
from quda_b200 import lib as L

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _native_loaded():
    import torch
    assert torch.cuda.is_available(), "GPU tier needs a CUDA device"
    lib = L.load()
    before = lib.b200_launch_count()
    yield
    assert lib.b200_launch_count() > before, "no kernel from libquda_b200.so was launched"


@pytest.fixture(scope="module")
def gpu():
    return C.Tier(True)


@pytest.fixture(scope="module")
def twin():
    return C.Tier(False)


@pytest.mark.parametrize("field", list(C.BUILD_FIELDS))
@pytest.mark.parametrize("prec", [8, 4])
@pytest.mark.parametrize("shape", list(C.SHAPES))
def test_build(gpu, twin, shape, prec, field):
    X = C.SHAPES[shape]
    A, inv, tl, _ = C.check_build(gpu, X, prec, *C.BUILD_FIELDS[field])
    links, clover = C.BUILD_FIELDS[field]
    gauge = C.gauge_field(X, links, 11, prec)
    coeff = C.coeff_for(gauge, X, clover)
    again = gpu.build(gauge, X, prec, coeff)
    assert np.array_equal(again[0], A) and np.array_equal(again[1], inv) and again[2] == tl  # repeated calls
    if prec == 8:  # the site code rounds identically on the device and in the host twin
        tA, tinv, _ = twin.build(gauge, X, prec, coeff)
        assert np.array_equal(A, tA) and np.array_equal(inv, tinv)


@pytest.mark.parametrize("prec", [8, 4])
@pytest.mark.parametrize("name", list(C.FORCE_CASES))
def test_force(gpu, twin, name, prec):
    case = C.force_case(name, prec)
    got, _ = C.check_force(gpu, case)
    assert np.array_equal(gpu.force(case, prec), got)  # repeated calls
    if prec == 8:
        assert np.array_equal(twin.force(case, prec), got)


@pytest.mark.parametrize("prec", [8, 4])
@pytest.mark.parametrize("shape", ["4x6x8x10", "6x2x4x6"])
def test_border(gpu, twin, shape, prec):
    A, tl = C.check_border(gpu, C.SHAPES[shape], prec)
    if prec == 8:
        tA, ttl = C.check_border(twin, C.SHAPES[shape], prec)
        assert np.array_equal(A, tA)


def test_build_16x16x16x32_fp32(gpu):
    C.check_build(gpu, (16, 16, 16, 32), 4, "eps1e-2")
