"""GPU tier: BiCGStab on M x = b (b200_invert_bicgstab, lib/inv_bicgstab_quda.cpp) for the Wilson, clover and twisted-mass
operators.  The complex BLAS / reduction kernels have no ABI of their own: a product that pairs the wrong reals or
conjugates the wrong operand stops BiCGStab from converging on these non-Hermitian operators, and every solution is
checked on the host with the oracle's full operator, which catches an answer that converged to the wrong thing."""
import ctypes as C

import numpy as np
import pytest

import oracle
from common import CudaMem, Problem
from quda_b200 import dirac as DR
from quda_b200 import dslash as D
from quda_b200 import lib as L

pytestmark = pytest.mark.gpu
KAPPA = 0.12195
MU = 0.1
X8 = (8, 8, 8, 8)


def _ops(P, kind, matpc, kappa=KAPPA, mixed=False, stream=None, comm=None, Ps=None):
    kw = dict(clover=P.A, clover_inv=P.Ainv) if "clover" in kind else {}
    if kind.startswith("twistedmass"):
        kw["mu"] = MU
    precise = DR.Dirac(kind, P.U, kappa, matpc_type=matpc, stream=stream, comm=comm[8] if comm else None, **kw)
    if not mixed:
        return precise, None
    if Ps is None:
        Ps = Problem(P.X, 4, 12, CudaMem, clover=P.clover is not None, compressed=True, dynamic=True)
    kws = dict(clover=Ps.A, clover_inv=Ps.Ainv) if "clover" in kind else {}
    if kind.startswith("twistedmass"):
        kws["mu"] = MU
    sloppy = DR.Dirac(kind, Ps.U, kappa, matpc_type=matpc, stream=stream, comm=comm[4] if comm else None, **kws)
    sloppy._keep = Ps
    return precise, sloppy


def _full_residual(P, kind, x, b, kappa=KAPPA):
    """|M x - b| / |b| with the oracle's unpreconditioned operator, in float64"""
    x = x.astype(np.float64)
    if "clover" in kind:
        Mx = oracle.clover_mat(P.gauge, P.clover, x, P.X, kappa, 0)
    elif kind.startswith("twistedmass"):
        Mx = oracle.tm_mat(P.gauge, x, P.X, kappa, MU, 0)
    else:
        Mx = oracle.wil_mat(P.gauge, x, P.X, kappa, 0)
    return float(np.linalg.norm(Mx.astype(np.float64).ravel() - b.astype(np.float64).ravel()) / np.linalg.norm(b.ravel()))


def _solve(P, kind, matpc=DR.MATPC_EVEN_EVEN, mixed=False, kappa=KAPPA, tol=1e-10, stream=None, comm=None, seed=77):
    """invertQuda-style with the operator as given: prepare -> BiCGStab on M_pc -> reconstruct for the *pc types, BiCGStab on
    the full field otherwise; returns (solver result, host-verified full-system residual, solution, source)"""
    precise, sloppy = _ops(P, kind, matpc, kappa, mixed, stream, comm)
    b = P.spinor(seed=seed, nparity=2)
    bdev, xdev = P.to_dev(b, 2), P.empty(2)
    if precise.kind.endswith("pc"):
        src_p, sol_p = precise.prepare(xdev, bdev)
        pb = xdev.parity_bytes
        src = D.ColorSpinorField(xdev.buf[src_p * pb:(src_p + 1) * pb], P.X, P.prec)
        sol = D.ColorSpinorField(xdev.buf[sol_p * pb:(sol_p + 1) * pb], P.X, P.prec)
        rhs = P.empty()
        rhs.buf.copy_(src.buf)  # the source lives in x's other-parity half, which reconstruct overwrites
        sol.buf.zero_()
        res = DR.invert_bicgstab(precise, sloppy, sol, rhs, tol=tol, maxiter=2000)
        precise.reconstruct(xdev, bdev)
    else:
        res = DR.invert_bicgstab(precise, sloppy, xdev, bdev, tol=tol, maxiter=2000)
    x = P.to_host(xdev)
    return res, _full_residual(P, kind, x, b, kappa), x, b


CASES = [
    ("wilsonpc", dict(), DR.MATPC_EVEN_EVEN),
    ("wilsonpc", dict(), DR.MATPC_ODD_ODD_ASYMMETRIC),
    ("cloverpc", dict(clover=True, compressed=True, dynamic=True), DR.MATPC_EVEN_EVEN),
    ("cloverpc", dict(clover=True, compressed=False, dynamic=False), DR.MATPC_EVEN_EVEN),
    ("cloverpc", dict(clover=True, compressed=False, dynamic=False), DR.MATPC_ODD_ODD_ASYMMETRIC),
    ("cloverpc", dict(clover=True, compressed=True, dynamic=True), DR.MATPC_EVEN_EVEN_ASYMMETRIC),
    ("twistedmasspc", dict(), DR.MATPC_EVEN_EVEN),
    ("twistedmasspc", dict(), DR.MATPC_ODD_ODD_ASYMMETRIC),
]


@pytest.mark.parametrize("mixed", [False, True], ids=["fp64", "fp64-fp32"])
@pytest.mark.parametrize("kind,pkw,matpc", CASES, ids=[f"{k}-{'dyn' if p.get('dynamic') else ('static' if p else 'plain')}-matpc{m}"
                                                      for k, p, m in CASES])
def test_bicgstab_preconditioned_system(kind, pkw, matpc, mixed):
    P = Problem(X8, 8, 18, CudaMem, **pkw)
    res, true_res, x, _ = _solve(P, kind, matpc, mixed)
    assert np.isfinite(x).all()
    assert res.iter < 2000 and res.true_res < 5e-10, (res.iter, res.true_res)
    assert true_res < 1e-8, true_res
    if mixed:
        assert res.reliable_updates >= 1, res.reliable_updates


@pytest.mark.parametrize("kind", ["wilson", "clover"])
def test_bicgstab_full_system(kind):
    P = Problem(X8, 8, 18, CudaMem, clover=kind == "clover", compressed=True, dynamic=True)
    res, true_res, _, _ = _solve(P, kind)
    assert res.iter < 2000 and res.true_res < 5e-10, (res.iter, res.true_res)
    assert true_res < 1e-8, true_res


def test_bicgstab_trivial_system():
    """kappa = 0: M_pc = 1.  rho = <r0, r> and <r0, M p> are the same sum, so alpha = 1 exactly, s = 0, |t|^2 = 0 gives
    omega = 0 without a breakdown, and the solve ends after one iteration with x == b"""
    P = Problem(X8, 8, 18, CudaMem)
    res, _, x, b = _solve(P, "wilsonpc", kappa=0.0)
    assert res.iter == 1, res.iter
    assert res.reliable_updates == 0
    assert res.true_res == 0.0, res.true_res
    # the native order is a rotated gamma basis, so compare with b as the device holds it
    b_dev = P.to_host(P.to_dev(b, 2))
    assert np.isfinite(x).all() and np.array_equal(x, b_dev)
    assert _full_residual(P, "wilsonpc", x, b_dev, kappa=0.0) == 0.0


@pytest.mark.parametrize("mixed", [False, True])
def test_bicgstab_on_a_non_blocking_stream(mixed):
    """every kernel on the operator's stream, while the default stream is kept busy; the host follows one iteration behind"""
    import torch
    P = Problem(X8, 8, 18, CudaMem, clover=True, compressed=True, dynamic=True)
    side = torch.cuda.Stream()
    junk = torch.empty(64 << 20, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    for _ in range(20):
        junk.add_(1.0)
    with torch.cuda.stream(side):
        res, true_res, _, _ = _solve(P, "cloverpc", mixed=mixed, stream=side.cuda_stream)
        side.synchronize()
    assert res.iter < 2000 and res.true_res < 5e-10, (res.iter, res.true_res)
    assert true_res < 1e-8, true_res
    assert res.host_syncs <= res.iter + 4 * (res.reliable_updates + 2), (res.host_syncs, res.iter, res.reliable_updates)


def test_bicgstab_is_bit_reproducible():
    P = Problem(X8, 8, 18, CudaMem, clover=True, compressed=True, dynamic=True)
    a = _solve(P, "cloverpc", mixed=True)
    b = _solve(P, "cloverpc", mixed=True)
    assert a[0].iter == b[0].iter and a[0].true_res == b[0].true_res
    assert np.array_equal(a[2], b[2])


def test_bicgstab_self_partitioned():
    """one GPU that is its own neighbour in every dimension: every Dslash of the solve goes through pack + ghost + exterior,
    one halo exchange per precision"""
    from quda_b200 import comm
    P = Problem(X8, 8, 12, CudaMem, clover=True, compressed=True, dynamic=True)
    grid = comm.ProcessGrid((1, 1, 1, 1), 0)
    exs = {p: comm.HaloExchange(grid, P.X, p, mode="self") for p in (8, 4)}
    css = {p: e.comm_struct() for p, e in exs.items()}
    res, true_res, _, _ = _solve(P, "cloverpc", mixed=True, comm=css)
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
