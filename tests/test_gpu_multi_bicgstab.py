"""GPU tier, >= 2 GPUs on one box: BiCGStab to 1e-10 on a lattice split over 2 GPUs (clover, double / single mixed precision
with reliable updates), once with the complex scalars all-reduced in the reduction kernels through the NVLink mailboxes and
once through the host callback.  Skipped on single-GPU boxes."""
import pytest
import torch
import torch.multiprocessing as mp

from test_dist_gloo import _free_port

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")]


@pytest.mark.parametrize("allreduce", ["nvlink", "callback"])
def test_two_gpu_bicgstab_host_verified(allreduce):
    from bicgstab_worker import bicgstab_worker
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=bicgstab_worker, args=(r, 2, port, (1, 1, 1, 2), (8, 8, 8, 8), q, allreduce)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        res = [q.get(timeout=900) for _ in procs]
        for p in procs:
            p.join(timeout=120)
            assert p.exitcode == 0
    finally:  # never leave a rank behind on the GPUs
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(timeout=30)
    iters = {r[1] for r in res}
    assert len(iters) == 1, res  # every rank takes the same decisions from the same global sums
    for rank, it, rel_updates, solver_res, true_res, timed_out in res:
        assert not timed_out
        assert it < 3000 and solver_res < 5e-10, (it, solver_res)
        assert true_res < 1e-8, true_res
        assert rel_updates >= 1
