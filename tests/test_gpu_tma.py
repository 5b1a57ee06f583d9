"""GPU tier (-m gpu): the TMA-staged marching kernel (quda_b200/csrc/tma_kernel.cuh: cp.async.bulk.tensor box loads,
mbarrier producer/consumer pipeline) through the C ABI against the CPU oracle.  B200_TMA=2 makes the library fail
instead of silently falling back to the gather kernel, so every case below is a real TMA launch."""
import pytest

import ops
import oracle
from common import CudaMem, Problem, assert_close
from quda_b200 import dslash as D
from quda_b200 import lib as L

pytestmark = pytest.mark.gpu


@pytest.fixture
def tma(monkeypatch):
    import torch
    assert torch.cuda.is_available(), "GPU tier needs a CUDA device"
    monkeypatch.setenv("B200_TMA", "2")
    lib = L.load()
    before = lib.b200_launch_count()
    yield monkeypatch
    assert lib.b200_launch_count() > before, "no kernel from libquda_b200.so was launched"


@pytest.mark.parametrize("X,prec,recon", [((16, 4, 4, 4), 4, 12), ((16, 8, 4, 6), 4, 12), ((8, 4, 8, 4), 4, 8),
                                          ((32, 4, 4, 4), 4, 18), ((16, 4, 8, 4), 8, 12), ((16, 4, 4, 6), 8, 18),
                                          ((8, 6, 10, 4), 8, 8), ((48, 2, 2, 4), 4, 12), ((16, 16, 16, 16), 4, 12),
                                          ((16, 16, 16, 16), 8, 12)])
def test_tma_wilson_dslash(tma, X, prec, recon):
    dev = ops.check_wilson_dslash(CudaMem, None, prec, recon, X)
    if prec == 8:
        assert dev <= 1e-12


@pytest.mark.parametrize("links", [-1, 0, 2, 3, 4])
@pytest.mark.parametrize("grid", [1, 3, 37, 148, 1000])
def test_tma_pipeline_depths_and_work_ranges(tma, links, grid):
    ops.check_tma_work_ranges(CudaMem, None, tma, links, grid)


@pytest.mark.parametrize("prefetch", [2, 3, 4])
@pytest.mark.parametrize("rings", ["4 2", "5 2", "6 3", "8 4"])
@pytest.mark.parametrize("grid", [5, 148])
def test_tma_register_stream_links(tma, prefetch, rings, grid):
    ops.check_tma_register_stream_links(CudaMem, None, tma, prefetch, rings, grid)


@pytest.mark.parametrize("l2pf", [-1, 1, 2, 5])
def test_tma_l2_prefetch_lookahead(tma, l2pf):
    ops.check_tma_l2_prefetch_lookahead(CudaMem, None, tma, l2pf)


@pytest.mark.parametrize("tile", ["1 1", "2 1", "1 2", "4 2", "2 4", "4 4", "8 1"])
def test_tma_tiles(tma, tile):
    ops.check_tma_tiles(CudaMem, None, tma, tile)


@pytest.mark.parametrize("prec,recon", [(8, 18), (8, 12), (4, 12), (4, 8)])
def test_tma_xpay_fullfield(tma, prec, recon):
    ops.check_xpay_fullfield(CudaMem, None, prec, recon, X=(8, 4, 4, 6))


@pytest.mark.parametrize("prec", [8, 4])
@pytest.mark.parametrize("compressed,dynamic", [(True, True), (False, False)])
def test_tma_clover(monkeypatch, prec, compressed, dynamic):
    monkeypatch.setenv("B200_TMA", "1")
    ops.check_clover(CudaMem, None, prec, 12, compressed, dynamic, X=(8, 4, 6, 4))


def test_tma_matches_gather_kernel_bitwise(monkeypatch):
    """same arithmetic, operation for operation: the TMA kernel and the gather kernel must agree bit for bit"""
    import torch
    X = (16, 8, 8, 8)
    P = Problem(X, 4, 12, CudaMem)
    s = P.to_dev(P.spinor(seed=9))
    outs = []
    for mode in ("0", "2"):
        monkeypatch.setenv("B200_TMA", mode)
        out = P.empty()
        D.ApplyWilson(out, s, P.U, 0.0, None, 0, 0)
        torch.cuda.synchronize()
        outs.append(out.buf.clone())
    assert torch.equal(outs[0], outs[1])


def test_tma_32cubed_fp32_recon12_vs_oracle(tma):
    """BASELINE config 2 at full size through the TMA kernel"""
    from quda_b200 import fields as F
    X = (32, 32, 32, 32)
    gauge = oracle.random_gauge(X, 4, seed=137)
    s = oracle.random_spinor(X, 4, seed=5)
    U = D.load_gauge(gauge, X, 4, 12, t_boundary=-1)
    out = D.ColorSpinorField(CudaMem.empty(F.spinor_bytes(X, 4)), X, 4, 1)
    D.ApplyWilson(out, D.ColorSpinorField(CudaMem.put(F.spinor_to_native(s, 4)), X, 4, 1), U, 0.0, None, 0, 0)
    CudaMem.sync()
    got = F.spinor_from_native(CudaMem.get(out.buf), 32 ** 4 // 2, 4)
    assert_close(oracle.wil_dslash(gauge, s, X, 0, 0), got, 4, 12, "32^4 fp32 recon-12 TMA vs oracle")
