"""GPU tier, >= 2 GPUs on one box: multi-shift CG on a clover-PC lattice split over 2 GPUs (double / single mixed precision
with reliable updates and refinement), once with the scalars all-reduced in the reduction kernels through the NVLink
mailboxes and once through the host callback; every shift is checked on the global lattice.  Skipped on single-GPU boxes."""
import pytest
import torch

from dist_worker import run_ranks, solver_worker

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")]


@pytest.mark.parametrize("allreduce", ["nvlink", "callback"])
def test_two_gpu_multishift_host_verified(allreduce):
    res = run_ranks(solver_worker, 2, ((1, 1, 1, 2), (8, 8, 8, 8), "multishift", "cloverpc", True, allreduce), timeout=900)
    # every rank takes the same decisions from the same global sums
    assert len({(r["iter"], tuple(r["iter_offset"]), tuple(r["refine_iter"])) for r in res}) == 1, res
    for r in res:
        assert not r["timed_out"]
        assert 0 < r["iter"] < 3000, r["iter"]
        assert r["reliable_updates"] >= 1
        assert all(v <= 1e-10 for v in r["true_res_offset"]), r["true_res_offset"]
        assert all(v < 1e-8 for v in r["host_true_res"]), r["host_true_res"]
