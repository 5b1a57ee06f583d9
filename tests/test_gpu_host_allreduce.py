"""GPU tier: CG and BiCGStab with the host-callback all-reduce (the path of boxes without NVLink mailboxes) on one GPU.
A self-partitioned exchange with an identity callback and no mailbox ranks makes every global sum of the solve go through
the host, so the path is checked here against the default device-finalised one on the same system."""
import numpy as np
import pytest

from common import CudaMem, Problem
from solvers import X8, self_exchanges, set_host_allreduce, solve

pytestmark = pytest.mark.gpu
KIND = "cloverpc"
# reductions per iteration that wait on the host with the callback: CG <p, Ap> and |r|^2; BiCGStab K1, K3 and K4
HOST_WAITS = {"cg": 2, "bicgstab": 3}


@pytest.mark.parametrize("mixed", [False, True], ids=["fp64", "fp64-fp32"])
@pytest.mark.parametrize("solver", ["cg", "bicgstab"])
def test_host_allreduce_matches_the_device_path(solver, mixed):
    P = Problem(X8, 8, 12, CudaMem, clover=True, compressed=True, dynamic=True)
    exs, css = self_exchanges(P.X)
    out = {}
    for callback in (False, True):
        set_host_allreduce(css, callback)
        res, true_res, x, _ = solve(P, KIND, solver, mixed=mixed, comm=css)
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
