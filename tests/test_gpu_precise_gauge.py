"""GPU tier of the per-element bounds of tests/precise_gauge.py: the gauge force, the link update, the momentum action
and the plaquette of libquda_b200.so on the cases of the CPU tier, bit for bit against the host twin in fp64 and fp32
(gauge.h rounds only through fma_rn / mul_rn, IEEE division and sqrt, so both precisions give the same bits on the
device and on the host), repeated calls bit-identical (the sums on 512 and on 135 CTA partials per parity included),
and the in-place update on every special spectrum."""
import numpy as np
import pytest

import gauge_cases as G
import precise_gauge_cases as C
from gauge_twin import gauge_twin
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
    return G.Runner(L.load(), "b200", dev=True)


@pytest.fixture(scope="module")
def twin():
    return G.Runner(gauge_twin(), "twin")


@pytest.mark.parametrize("links", C.LINKS)
@pytest.mark.parametrize("prec", [8, 4])
@pytest.mark.parametrize("shape", list(C.SHAPES))
def test_force_links(gpu, twin, shape, prec, links):
    X = C.SHAPES[shape]
    got, _, _ = C.check_force(gpu, X, prec, links, "gauss", "plaq+rect", C.EB3["pos"])
    again, _, _ = C.check_force(gpu, X, prec, links, "gauss", "plaq+rect", C.EB3["pos"])
    assert C.same_bits(got, again), "repeated calls differ"
    assert C.same_bits(got, C.check_force(twin, X, prec, links, "gauss", "plaq+rect", C.EB3["pos"])[0])


@pytest.mark.parametrize("eb3", list(C.EB3))
@pytest.mark.parametrize("prec", [8, 4])
@pytest.mark.parametrize("paths", C.PATHS)
def test_force_paths(gpu, twin, paths, prec, eb3):
    X = C.SHAPES["6x2x4x6"] if paths == "table-limit" else C.SHAPES["4x6x8x10"]
    args = (X, prec, "mixed", "spread", paths, C.EB3[eb3], True)
    got = C.check_force(gpu, *args)[0]
    assert C.same_bits(got, C.check_force(twin, *args)[0])


@pytest.mark.parametrize("links", C.LINKS)
@pytest.mark.parametrize("prec", [8, 4])
@pytest.mark.parametrize("mom", C.MOMS)
def test_force_moms(gpu, twin, mom, prec, links):
    args = (C.SHAPES["2x4x6x4"], prec, links, mom, "symanzik48", C.EB3["neg"], True)
    assert C.same_bits(C.check_force(gpu, *args)[0], C.check_force(twin, *args)[0])


UPDATE_RUNS = [(0.7, False), (0.7, True), (-0.4, False)]  # (dt, conj_mom)


@pytest.mark.parametrize("run", range(len(UPDATE_RUNS)))
@pytest.mark.parametrize("prec", [8, 4])
@pytest.mark.parametrize("kind", C.SPECTRA)
def test_update(gpu, twin, kind, prec, run):
    dt, conj = UPDATE_RUNS[run]
    X = C.SHAPES["6x2x4x6"]
    for exact in ([True, False] if kind in C.SMALL else [True]):
        got, _, _, gauge, mom = C.check_update(gpu, X, prec, kind, dt, conj, exact)
        assert C.same_bits(got, gpu.update(gauge, mom, X, dt, conj, exact, prec)), "repeated calls differ"
        assert C.same_bits(got, gpu.update(gauge, mom, X, dt, conj, exact, prec, in_place=True)), "in place differs"
        assert C.same_bits(got, twin.update(gauge, mom, X, dt, conj, exact, prec)), "the twin differs"


@pytest.mark.parametrize("prec", [8, 4])
@pytest.mark.parametrize("shape", list(C.SUM_SHAPES))
def test_sums(gpu, twin, shape, prec):
    X = C.SUM_SHAPES[shape]
    i = list(C.SUM_SHAPES).index(shape)
    S, _, _, mom = C.check_mom_action(gpu, X, prec, C.MOMS[i % len(C.MOMS)])
    assert S == gpu.mom_action(mom, X, prec), "repeated calls differ"
    assert S == twin.mom_action(mom, X, prec), "the twin differs"
    links = C.LINKS[i % len(C.LINKS)]
    pl, _, _ = C.check_plaquette(gpu, X, prec, links)
    gauge = C.links(X, links, seed=31).astype(np.float64 if prec == 8 else np.float32)
    assert pl == gpu.plaquette(gauge, X, prec), "repeated calls differ"
    assert pl == twin.plaquette(gauge, X, prec), "the twin differs"
