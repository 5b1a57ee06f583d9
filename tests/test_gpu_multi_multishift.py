"""GPU tier, >= 2 GPUs on one box: multi-shift CG on a clover-PC lattice split over 2 GPUs (double / single mixed precision
with reliable updates and refinement), once with the scalars all-reduced in the reduction kernels through the NVLink
mailboxes and once through the host callback; every shift is checked on the global lattice.  Skipped on single-GPU boxes."""
import pytest
import torch
import torch.multiprocessing as mp

from test_dist_gloo import _free_port

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")]


@pytest.mark.parametrize("allreduce", ["nvlink", "callback"])
def test_two_gpu_multishift_host_verified(allreduce):
    from multishift_worker import multishift_worker
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=multishift_worker, args=(r, 2, port, (1, 1, 1, 2), (8, 8, 8, 8), q, allreduce))
             for r in range(2)]
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
    # every rank takes the same decisions from the same global sums
    assert len({(r[1], tuple(r[2]), tuple(r[3])) for r in res}) == 1, res
    for rank, it, iter_offset, refine, rel_updates, solver_res, true_res, timed_out in res:
        assert not timed_out
        assert 0 < it < 3000, it
        assert rel_updates >= 1
        assert all(r <= 1e-10 for r in solver_res), solver_res
        assert all(r < 1e-8 for r in true_res), true_res
