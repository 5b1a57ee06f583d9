"""CPU tier: the TMA-staged marching kernel's plan / tensor-map / ring-slot / shared-memory-offset logic
(quda_b200/csrc/tma.h), emulated by the host twin (tests/hosttwin/tma_emu.h) against the oracle.

B200_TMA=2 makes the twin FAIL if the TMA path does not serve the shape, so every case below really walks the
emulated pipeline: box loads interpreted from the tensor-map descriptions, producer program replayed against slot
ownership (overwriting a live slot, reading a released one -- it is poisoned with NaNs -- or a state where neither
producer nor consumers can advance all fail the test)."""
import pytest

import ops
from common import HostMem, Problem, twin_backend


@pytest.fixture
def tma(monkeypatch):
    monkeypatch.setenv("B200_TMA", "2")
    return monkeypatch


@pytest.mark.parametrize("X,prec,recon", [((16, 4, 4, 4), 4, 12), ((16, 8, 4, 6), 4, 12), ((8, 4, 8, 4), 4, 8),
                                          ((32, 4, 4, 4), 4, 18), ((16, 4, 8, 4), 8, 12), ((16, 4, 4, 6), 8, 18),
                                          ((8, 6, 10, 4), 8, 8), ((48, 2, 2, 4), 4, 12)])
def test_tma_wilson_dslash(tma, X, prec, recon):
    ops.check_wilson_dslash(HostMem, twin_backend(), prec, recon, X)


@pytest.mark.parametrize("links", [-1, 0, 2, 3, 4])
@pytest.mark.parametrize("grid", [1, 3, 7, 37, 148, 1000])
def test_tma_pipeline_depths_and_work_ranges(tma, links, grid):
    ops.check_tma_work_ranges(HostMem, twin_backend(), tma, links, grid)


@pytest.mark.parametrize("prefetch", [2, 3, 4])
@pytest.mark.parametrize("rings", ["4 2", "5 2", "6 3", "8 4"])
@pytest.mark.parametrize("grid", [5, 148])
def test_tma_register_stream_links(tma, prefetch, rings, grid):
    ops.check_tma_register_stream_links(HostMem, twin_backend(), tma, prefetch, rings, grid)


@pytest.mark.parametrize("l2pf", [-1, 1, 2, 5])
def test_tma_l2_prefetch_lookahead(tma, l2pf):
    ops.check_tma_l2_prefetch_lookahead(HostMem, twin_backend(), tma, l2pf)


@pytest.mark.parametrize("tile", ["1 1", "2 1", "1 2", "4 2", "2 4", "4 4", "8 1"])
def test_tma_tiles(tma, tile):
    ops.check_tma_tiles(HostMem, twin_backend(), tma, tile)


@pytest.mark.parametrize("prec,recon", [(8, 18), (8, 12), (4, 12), (4, 8)])
def test_tma_xpay_fullfield(tma, prec, recon):
    ops.check_xpay_fullfield(HostMem, twin_backend(), prec, recon, X=(8, 4, 4, 6))


@pytest.mark.parametrize("prec", [8, 4])
@pytest.mark.parametrize("compressed,dynamic", [(True, True), (False, False)])
def test_tma_clover(monkeypatch, prec, compressed, dynamic):
    # B200_TMA=1: ApplyClover and the dagger-xpay corner are not TMA launches, they take the gather path
    monkeypatch.setenv("B200_TMA", "1")
    ops.check_clover(HostMem, twin_backend(), prec, 12, compressed, dynamic, X=(8, 4, 6, 4))


def test_tma_unserved_shapes_fall_back(monkeypatch):
    """half precision and odd extents are not served: B200_TMA=1 silently uses the gather kernel, results unchanged"""
    monkeypatch.setenv("B200_TMA", "1")
    be = twin_backend()
    for X, prec, recon in (((4, 4, 4, 4), 2, 12), ((4, 6, 2, 2), 4, 12)):
        P = Problem(X, prec, recon, HostMem)
        ops.wilson_vs_oracle(P, be, P.spinor(seed=2), 0, 0, f"fallback X={X}")
