"""GPU tier: the case bodies of tests/ops.py (ops.check_*, which the CPU tier runs on the host twin) through
libquda_b200.so -- xpay / dagger / full fields, clover variants, multi-RHS batches, twisted mass and the
self-partitioned halo path (pack kernel -> ghost buffers -> interior + fused exterior kernel) for the partition masks
dslash_ctest uses (tests/dslash_ctest.cpp:40-42,174-186) -- plus the self exchange with arrival flags."""
import numpy as np
import pytest

import oracle
import ops
from common import CudaMem, Problem, assert_close
from quda_b200 import comm, dslash as D

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("prec", [8, 4, 2])
@pytest.mark.parametrize("recon", [18, 12, 8])
def test_xpay_dagger_fullfield(prec, recon):
    ops.check_xpay_fullfield(CudaMem, None, prec, recon)


@pytest.mark.parametrize("prec", [8, 4, 2])
@pytest.mark.parametrize("compressed,dynamic", [(True, True), (False, False)])
def test_clover(prec, compressed, dynamic):
    ops.check_clover(CudaMem, None, prec, 12, compressed, dynamic)


def test_clover_half_recon8_config3():
    """BASELINE config 3: clover-preconditioned Dslash, half precision, recon-8 (tolerance 1e-3 x 10)"""
    ops.check_clover(CudaMem, None, 2, 8, True, True, X=(8, 8, 8, 8))


@pytest.mark.parametrize("comm_dim", [(1, 0, 0, 0), (0, 1, 0, 0), (0, 0, 1, 0), (0, 0, 0, 1), (1, 1, 0, 0), (0, 0, 1, 1), (1, 1, 1, 1)])
@pytest.mark.parametrize("prec,recon", [(8, 18), (4, 12), (2, 8)])
def test_partitioned_wilson(prec, recon, comm_dim):
    ops.check_partitioned(CudaMem, None, prec, recon, comm_dim, X=(4, 6, 4, 8), xpay=True, dagger=1)


@pytest.mark.parametrize("op", ["clover_pc", "clover"])
def test_partitioned_clover(op):
    ops.check_partitioned(CudaMem, None, 4, 12, (1, 1, 1, 1), op=op, xpay=True, clover_kw=dict(compressed=True, dynamic=True))


@pytest.mark.parametrize("prec,recon", [(8, 18), (4, 12), (2, 12)])
def test_self_exchange_with_arrival_flags(prec, recon):
    """The NVLink remote-write protocol on one GPU: the pack kernel raises sequence-numbered flags, the exterior
    kernel spins on them; ten back-to-back applications exercise the double-buffered ghost zones."""
    X = (8, 4, 4, 8)
    P = Problem(X, prec, recon, CudaMem)
    grid = comm.ProcessGrid((1, 1, 1, 1), 0)
    ex = comm.HaloExchange(grid, X, prec, mode="self")
    s = P.spinor(seed=1)
    ref = oracle.wil_dslash(P.gauge, s, X, 0, 0)
    din, out = P.to_dev(s), P.empty()
    for _ in range(10):
        comm.apply_wilson_distributed(ex, out, din, P.U, 0.0, None, 0, 0)
    assert_close(ref, P.to_host(out), prec, recon, "self exchange")
    assert not ex.timed_out()


@pytest.mark.parametrize("prec,recon", [(8, 18), (8, 12), (4, 18), (4, 12), (4, 8), (2, 12), (2, 8)])
@pytest.mark.parametrize("n_src", [2, 7, 8])
@pytest.mark.parametrize("flavour", ["thread", "auto"])
def test_multi_rhs_wilson(monkeypatch, prec, recon, n_src, flavour):
    """batched Dslash (the reference's cvector_ref form): oracle parity per source + bit-identity with the
    single-source kernel; thread flavour: 7 = one 4-batch, one 2-batch and the single-source tail (fp64: 2+2+2+1);
    "auto" = the library's default flavour for the precision"""
    monkeypatch.setenv("B200_MRHS_MODE", flavour)
    ops.check_multi_rhs(CudaMem, None, prec, recon, n_src, xpay=(n_src == 7), dagger=n_src % 2)


@pytest.mark.parametrize("op", ["clover_pc", "clover"])
@pytest.mark.parametrize("prec", [8, 4, 2])
def test_multi_rhs_clover(monkeypatch, op, prec):
    monkeypatch.setenv("B200_MRHS_MODE", "thread")
    ops.check_multi_rhs(CudaMem, None, prec, 12, 4, op=op, xpay=True)


def test_multi_rhs_full_fields_and_fallback():
    ops.check_multi_rhs(CudaMem, None, 4, 12, 4, xpay=True, nparity=2)
    ops.check_multi_rhs(CudaMem, None, 8, 18, 1, comm_dim=(1, 0, 0, 1), X=(4, 4, 4, 4))


def test_multi_rhs_16cubed_tiles():
    """a lattice large enough for the production tile shapes (full x rows), 16 sources = QUDA_MAX_MULTI_RHS"""
    ops.check_multi_rhs(CudaMem, None, 4, 12, 16, X=(16, 8, 8, 8))
    ops.check_multi_rhs(CudaMem, None, 2, 8, 4, X=(16, 8, 8, 8), tile=(8, 8, 1, 1))


@pytest.mark.parametrize("prec,recon", [(8, 18), (4, 12), (4, 8), (2, 12), (2, 8)])
@pytest.mark.parametrize("n_src,cta_sources,l1,cfg", [(2, 0, 1, 0), (7, 2, 1, 1), (8, 0, 0, 0), (16, 3, 1, 2), (8, 0, 1, 1)])
def test_multi_rhs_cta_flavour(monkeypatch, prec, recon, n_src, cta_sources, l1, cfg):
    """B200_MRHS_MODE=cta: one thread per (site, source), the sources of a site share a CTA and the links through L1;
    cfg = occupancy configuration (register budget) of the kernel"""
    monkeypatch.setenv("B200_MRHS_MODE", "cta")
    monkeypatch.setenv("B200_MRHS_CTA_SOURCES", str(cta_sources))
    monkeypatch.setenv("B200_MRHS_L1", str(l1))
    monkeypatch.setenv("B200_MRHS_CTA_CFG", str(cfg))
    ops.check_multi_rhs(CudaMem, None, prec, recon, n_src, xpay=(n_src == 7), dagger=n_src % 2, X=(16, 4, 4, 4),
                        tile=(8, 2, 1, 1))


def test_multi_rhs_cta_flavour_clover_and_full(monkeypatch):
    monkeypatch.setenv("B200_MRHS_MODE", "cta")
    ops.check_multi_rhs(CudaMem, None, 4, 12, 3, op="clover_pc", xpay=True)
    ops.check_multi_rhs(CudaMem, None, 2, 12, 3, op="clover", xpay=True, tile=(2, 2, 1, 1))
    ops.check_multi_rhs(CudaMem, None, 4, 12, 4, xpay=True, nparity=2, tile=(2, 2, 2, 2))


@pytest.mark.parametrize("prec,recon", [(8, 18), (4, 12), (4, 8), (2, 12)])
def test_twisted_mass(prec, recon):
    """degenerate twisted mass (ApplyTwistedMass / ApplyTwistedMassPreconditioned + the DiracTwistedMassPC composition,
    all four matpc types x dagger) against the oracle's tm_dslash / tm_mat / tm_matpc"""
    ops.check_twisted_mass(CudaMem, None, prec, recon)


def test_twisted_mass_partitioned():
    ops.check_twisted_mass(CudaMem, None, 4, 12, X=(4, 4, 4, 4), comm_dim=(1, 0, 1, 1))
