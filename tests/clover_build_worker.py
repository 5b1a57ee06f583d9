"""Multi-rank worker of the clover construction tests: every rank extends its block of a global gauge field by a depth-1
halo (comm.extend_gauge), computes its clover term and tr log A, and reports the deviation from the GLOBAL reference
(tests/clover_build_ref.py).  Mode "host": gloo + host twin (CPU tier); "gpu": NCCL, one GPU per rank, libquda_b200.so,
with trlog all-reduced by dslash.compute_clover_field (GPU tier)."""
import os

import numpy as np

from dist_worker import _join, _leave

KAPPA, CSW = 0.12195, 1.4


def worker(rank, world, port, q, grid_dims, Xl, mode="host"):
    os.environ["OMP_NUM_THREADS"] = "2"
    dist = _join(rank, world, port, "gloo" if mode == "host" else "nccl")
    import torch

    import clover_build_ref as R
    import oracle
    from quda_b200 import comm
    from quda_b200 import dslash as D
    grid = comm.ProcessGrid(grid_dims, rank)
    Xg = [Xl[d] * grid_dims[d] for d in range(4)]
    gauge = oracle.random_gauge(Xg, 8, seed=137)  # same global field on every rank
    ref = R.compute_clover(gauge, Xg, KAPPA * CSW)
    want = comm.local_slice(ref, Xg, Xl, grid.coords, "clover")
    local = comm.local_slice(gauge, Xg, Xl, grid.coords, "gauge")
    if mode == "host":
        from clover_twin import clover_twin
        be = clover_twin()
        got = np.zeros((int(np.prod(Xl)), 2, 36))
        D.compute_clover(got, comm.extend_gauge(grid, local, Xl, dist), Xl, grid.comm_dim(), 8, KAPPA * CSW, backend=be)
        t = torch.tensor(D.clover_invert(None, got, Xl, 8, backend=be), dtype=torch.float64)
        dist.all_reduce(t)
        trlog = t.tolist()
    else:
        dev_local = torch.from_numpy(local).cuda()
        packed = torch.empty((int(np.prod(Xl)), 2, 36), dtype=torch.float64, device="cuda")
        D.compute_clover(packed, comm.extend_gauge(grid, dev_local, Xl, dist), Xl, grid.comm_dim(), 8, KAPPA * CSW)
        got = packed.cpu().numpy()
        _, _, trlog = D.compute_clover_field(local, Xl, 8, KAPPA, CSW, grid=grid, dist=dist)
    dev = float(np.abs(got - want).max())
    _leave(dist, q, {"rank": rank, "dev": dev, "trlog": list(trlog), "trlog_ref": R.trlog(ref).tolist()})
