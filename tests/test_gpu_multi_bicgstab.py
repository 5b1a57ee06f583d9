"""GPU tier, >= 2 GPUs on one box: BiCGStab to 1e-10 on a lattice split over 2 GPUs (clover, double / single mixed precision
with reliable updates), once with the complex scalars all-reduced in the reduction kernels through the NVLink mailboxes and
once through the host callback.  Skipped on single-GPU boxes."""
import pytest
import torch

from dist_worker import run_ranks, solver_worker

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")]


@pytest.mark.parametrize("allreduce", ["nvlink", "callback"])
def test_two_gpu_bicgstab_host_verified(allreduce):
    res = run_ranks(solver_worker, 2, ((1, 1, 1, 2), (8, 8, 8, 8), "bicgstab", "cloverpc", True, allreduce), timeout=900)
    iters = {r["iter"] for r in res}
    assert len(iters) == 1, res  # every rank takes the same decisions from the same global sums
    for r in res:
        assert not r["timed_out"]
        assert r["iter"] < 3000 and r["true_res"] < 5e-10, (r["iter"], r["true_res"])
        assert r["host_true_res"] < 1e-8, r["host_true_res"]
        assert r["reliable_updates"] >= 1
