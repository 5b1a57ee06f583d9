"""GPU tier: CG and BiCGStab with the host-callback all-reduce (the path of boxes without NVLink mailboxes) on one GPU.
A self-partitioned exchange with an identity callback and no mailbox ranks makes every global sum of the solve go through
the host, so the path is checked here against the default device-finalised one on the same system."""
import ctypes as C

import numpy as np
import pytest

from common import CudaMem, Problem
from quda_b200 import dirac as DR
from quda_b200 import dslash as D
from quda_b200 import lib as L
from test_gpu_bicgstab import X8, _full_residual, _ops

pytestmark = pytest.mark.gpu
KIND = "cloverpc"
# reductions per iteration that wait on the host with the callback: CG <p, Ap> and |r|^2; BiCGStab K1, K3 and K4
HOST_WAITS = {"cg": 2, "bicgstab": 3}


def _solve(P, solver, mixed, css):
    """prepare -> CG on M_pc^dag M_pc (source M_pc^dag src) or BiCGStab on M_pc -> reconstruct; returns (solver result,
    host-verified full-system residual, solution)"""
    precise, sloppy = _ops(P, KIND, DR.MATPC_EVEN_EVEN, mixed=mixed, comm=css)
    b = P.spinor(seed=77, nparity=2)
    bdev, xdev = P.to_dev(b, 2), P.empty(2)
    src_p, sol_p = precise.prepare(xdev, bdev)
    pb = xdev.parity_bytes
    src = D.ColorSpinorField(xdev.buf[src_p * pb:(src_p + 1) * pb], P.X, P.prec)
    sol = D.ColorSpinorField(xdev.buf[sol_p * pb:(sol_p + 1) * pb], P.X, P.prec)
    rhs = P.empty()
    if solver == "cg":
        precise.Mdag(rhs, src)
    else:
        rhs.buf.copy_(src.buf)  # the source lives in x's other-parity half, which reconstruct overwrites
    sol.buf.zero_()
    invert = DR.invert_cg if solver == "cg" else DR.invert_bicgstab
    res = invert(precise, sloppy, sol, rhs, tol=1e-10, maxiter=2000)
    precise.reconstruct(xdev, bdev)
    x = P.to_host(xdev)
    return res, _full_residual(P, KIND, x, b), x


@pytest.mark.parametrize("mixed", [False, True], ids=["fp64", "fp64-fp32"])
@pytest.mark.parametrize("solver", ["cg", "bicgstab"])
def test_host_allreduce_matches_the_device_path(solver, mixed):
    from quda_b200 import comm
    P = Problem(X8, 8, 12, CudaMem, clover=True, compressed=True, dynamic=True)
    grid = comm.ProcessGrid((1, 1, 1, 1), 0)
    exs = {p: comm.HaloExchange(grid, P.X, p, mode="self") for p in (8, 4)}
    css = {p: e.comm_struct() for p, e in exs.items()}
    identity = L.ALLREDUCE_FN(lambda data, n, user: None)  # one rank: the global sum is the local one
    out = {}
    for callback in (False, True):
        for cs in css.values():
            assert cs.n_ranks == 0  # no mailboxes: with a callback set, every sum goes through it
            cs.allreduce_sum = C.cast(identity, C.c_void_p) if callback else None
        res, true_res, x = _solve(P, solver, mixed, css)
        assert np.isfinite(x).all()
        assert res.iter < 2000 and res.true_res < 5e-10, (callback, res.iter, res.true_res)
        assert true_res < 1e-8, (callback, true_res)
        bound = HOST_WAITS[solver] * res.iter + 4 * (res.reliable_updates + 2)
        assert res.host_syncs <= bound, (callback, res.host_syncs, res.iter, res.reliable_updates)
        assert not any(e.timed_out() for e in exs.values())
        out[callback] = (res, x)
    if mixed:
        return
    (dev, x_dev), (host, x_host) = out[False], out[True]
    if solver == "bicgstab":
        # both paths derive the scalars with the same function, and the done flag makes the iteration counts agree
        assert dev.iter == host.iter and dev.true_res == host.true_res, (dev.iter, host.iter, dev.true_res, host.true_res)
        assert np.array_equal(x_dev, x_host)
    else:
        # with the callback the host decides in the iteration that reached the tolerance; the device path one iteration late
        assert dev.iter == host.iter + 1, (dev.iter, host.iter)
