"""GPU worker of tests/test_gpu_batched_halo.py (run as a subprocess so that a device fault cannot take the rest of the GPU
tier with it): the batched multi-RHS halo (b200_pack_ghost_multi) on one GPU that is its own neighbour.
  1. PackGhostMulti + per-source Dslash on plain ghost buffers (arrival by stream order) -- ops.check_partitioned_multi,
     the case body the host twin runs in the CPU tier (tests/test_twin_ops.py::test_batched_halo_*);
  2. HaloExchange(mode="self", n_src=...): the arrival-counter protocol (one signal per face for the whole batch), batched
     and single exchanges interleaved on the same double-buffered slabs.
Prints one line per case and "ALL OK" at the end."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402

import oracle  # noqa: E402
import ops  # noqa: E402
from common import CudaMem, Problem, assert_close  # noqa: E402
from quda_b200 import comm  # noqa: E402


def main():
    for prec, recon, n_src, mask, kw in [
            (8, 18, 3, (0, 0, 0, 1), dict(xpay=True)),
            (4, 12, 8, (1, 1, 1, 1), dict(dagger=1)),
            (4, 8, 16, (0, 1, 1, 1), dict(xpay=True, aligned=False)),
            (2, 12, 5, (1, 0, 1, 0), dict()),
            (2, 8, 2, (0, 0, 1, 1), dict(xpay=True, dagger=1)),
            (4, 12, 4, (0, 1, 1, 1), dict(op="clover_pc", xpay=True, split="tiles", clover_kw=dict(compressed=True, dynamic=True))),
            (8, 12, 3, (1, 1, 0, 1), dict(op="clover", split="sites", clover_kw=dict(compressed=True, dynamic=True)))]:
        ops.check_partitioned_multi(CudaMem, None, prec, recon, mask, n_src, X=(4, 6, 4, 8), **kw)
        print("ok stream-order", prec, recon, n_src, mask, kw, flush=True)
    for prec, recon, n_src, dims in [(8, 18, 3, (0, 0, 0, 1)), (4, 12, 8, (0, 1, 1, 1)), (2, 12, 4, (1, 1, 1, 1))]:
        X = (8, 4, 4, 8)
        P = Problem(X, prec, recon, CudaMem)
        ex = comm.HaloExchange(comm.ProcessGrid((1, 1, 1, 1), 0), X, prec, mode="self", self_dims=dims, n_src=n_src)
        src = [P.spinor(seed=10 + i) for i in range(n_src)]
        dins, outs, one = [P.to_dev(s) for s in src], [P.empty() for _ in range(n_src)], P.empty()
        for rep in range(5):  # batched, batched, single, ... on the same two buffers
            comm.apply_wilson_distributed(ex, outs, dins, P.U, 0.0, None, 0, 0)
            if rep % 2:
                comm.apply_wilson_distributed(ex, one, dins[1], P.U, 0.0, None, 0, 0)
        for i in range(n_src):
            assert_close(oracle.wil_dslash(P.gauge, src[i], X, 0, 0), P.to_host(outs[i]), prec, recon, f"batched self exchange src {i}")
        assert np.array_equal(P.to_host(one), P.to_host(outs[1]))
        assert not ex.timed_out(), "a boundary kernel gave up waiting for the batch's arrival counter"
        print("ok arrival-counters", prec, recon, n_src, dims, flush=True)
    print("ALL OK", flush=True)


if __name__ == "__main__":
    main()
