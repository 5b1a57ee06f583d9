"""GPU tier: BiCGStab on M x = b (b200_invert_bicgstab, lib/inv_bicgstab_quda.cpp) for the Wilson, clover and twisted-mass
operators.  The complex BLAS / reduction kernels have no ABI of their own: a product that pairs the wrong reals or
conjugates the wrong operand stops BiCGStab from converging on these non-Hermitian operators, and every solution is
checked on the host with the oracle's full operator, which catches an answer that converged to the wrong thing."""
import ctypes as C

import numpy as np
import pytest

from common import CudaMem, Problem
from quda_b200 import dirac as DR
from quda_b200 import lib as L
from solvers import CASE_IDS, CASES, KAPPA, X8, busy_default_stream, full_residual, self_exchanges, solve

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("mixed", [False, True], ids=["fp64", "fp64-fp32"])
@pytest.mark.parametrize("kind,pkw,matpc", CASES, ids=CASE_IDS)
def test_bicgstab_preconditioned_system(kind, pkw, matpc, mixed):
    P = Problem(X8, 8, 18, CudaMem, **pkw)
    res, true_res, x, _ = solve(P, kind, "bicgstab", matpc, mixed)
    assert np.isfinite(x).all()
    assert res.iter < 2000 and res.true_res < 5e-10, (res.iter, res.true_res)
    assert true_res < 1e-8, true_res
    if mixed:
        assert res.reliable_updates >= 1, res.reliable_updates


@pytest.mark.parametrize("kind", ["wilson", "clover"])
def test_bicgstab_full_system(kind):
    P = Problem(X8, 8, 18, CudaMem, clover=kind == "clover", compressed=True, dynamic=True)
    res, true_res, _, _ = solve(P, kind, "bicgstab")
    assert res.iter < 2000 and res.true_res < 5e-10, (res.iter, res.true_res)
    assert true_res < 1e-8, true_res


def test_bicgstab_trivial_system():
    """kappa = 0: M_pc = 1.  rho = <r0, r> and <r0, M p> are the same sum, so alpha = 1 exactly, s = 0, |t|^2 = 0 gives
    omega = 0 without a breakdown, and the solve ends after one iteration with x == b"""
    P = Problem(X8, 8, 18, CudaMem)
    res, _, x, b = solve(P, "wilsonpc", "bicgstab", kappa=0.0)
    assert res.iter == 1, res.iter
    assert res.reliable_updates == 0
    assert res.true_res == 0.0, res.true_res
    # the native order is a rotated gamma basis, so compare with b as the device holds it
    b_dev = P.to_host(P.to_dev(b, 2))
    assert np.isfinite(x).all() and np.array_equal(x, b_dev)
    assert full_residual(P, "wilsonpc", x, b_dev, kappa=0.0) == 0.0


@pytest.mark.parametrize("mixed", [False, True])
def test_bicgstab_on_a_non_blocking_stream(mixed):
    """every kernel on the operator's stream, while the default stream is kept busy; the host follows one iteration behind"""
    P = Problem(X8, 8, 18, CudaMem, clover=True, compressed=True, dynamic=True)
    with busy_default_stream() as side:
        res, true_res, _, _ = solve(P, "cloverpc", "bicgstab", mixed=mixed, stream=side.cuda_stream)
    assert res.iter < 2000 and res.true_res < 5e-10, (res.iter, res.true_res)
    assert true_res < 1e-8, true_res
    assert res.host_syncs <= res.iter + 4 * (res.reliable_updates + 2), (res.host_syncs, res.iter, res.reliable_updates)


def test_bicgstab_is_bit_reproducible():
    P = Problem(X8, 8, 18, CudaMem, clover=True, compressed=True, dynamic=True)
    a = solve(P, "cloverpc", "bicgstab", mixed=True)
    b = solve(P, "cloverpc", "bicgstab", mixed=True)
    assert a[0].iter == b[0].iter and a[0].true_res == b[0].true_res
    assert np.array_equal(a[2], b[2])


def test_bicgstab_self_partitioned():
    """one GPU that is its own neighbour in every dimension: every Dslash of the solve goes through pack + ghost + exterior,
    one halo exchange per precision"""
    P = Problem(X8, 8, 12, CudaMem, clover=True, compressed=True, dynamic=True)
    exs, css = self_exchanges(P.X)
    res, true_res, _, _ = solve(P, "cloverpc", "bicgstab", mixed=True, comm=css)
    assert res.iter < 2000 and res.true_res < 5e-10, (res.iter, res.true_res)
    assert true_res < 1e-8, true_res
    assert res.reliable_updates >= 1
    assert not any(e.timed_out() for e in exs.values())


def test_bicgstab_argument_checks():
    lib = L.load()
    P = Problem((4, 4, 4, 4), 8, 18, CudaMem)
    op = DR.Dirac("wilsonpc", P.U, KAPPA)
    x, b = P.empty(), P.to_dev(P.spinor(seed=3))
    p = L.SolverParam()
    p.tol, p.maxiter = 1e-10, 10
    xd, bd = x.desc(), b.desc()
    assert lib.b200_invert_bicgstab(None, None, C.byref(xd), C.byref(bd), C.byref(p)) == -1
    assert b"null" in lib.b200_last_error()
    assert lib.b200_invert_bicgstab(op.h, None, C.byref(xd), C.byref(bd), None) == -1
    assert b"null" in lib.b200_last_error()

    def refused(sloppy, match, precise=op, xf=x, bf=b):
        with pytest.raises(L.B200Error, match=match):
            DR.invert_bicgstab(precise, sloppy, xf, bf, tol=1e-10, maxiter=10)

    Ph = Problem((4, 4, 4, 4), 2, 12, CudaMem)
    refused(DR.Dirac("wilsonpc", Ph.U, KAPPA), "double or single")
    Ps = Problem((4, 4, 4, 4), 4, 12, CudaMem)
    op4 = DR.Dirac("wilsonpc", Ps.U, KAPPA)
    refused(op, "more precise", precise=op4, xf=Ps.empty(), bf=Ps.to_dev(Ps.spinor(seed=3)))
    import torch
    side = torch.cuda.Stream()
    refused(DR.Dirac("wilsonpc", Ps.U, KAPPA, stream=side.cuda_stream), "share a stream")
    refused(None, "precision", xf=Ps.empty())
    refused(None, "precision", bf=Ps.to_dev(Ps.spinor(seed=3)))
