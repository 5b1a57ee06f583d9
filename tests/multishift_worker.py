"""Two-rank multi-shift CG worker: every rank owns one block of a global lattice, the C++ solver layer exchanges every Dslash
halo over NVLink and all-reduces the scalars either in the reduction kernels (NVLink mailboxes, B200_ALLREDUCE=nvlink) or
through the host callback (B200_ALLREDUCE=callback).  The solves are clover-PC (symmetric even-even), double with a
single-precision sloppy operator; each gathered x_j is verified on the GLOBAL lattice with the oracle's
M_pc^dag M_pc + sigma_j."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OFFSETS = [0.0, 1e-3, 1e-2, 0.1, 1.0, 10.0]


def multishift_worker(rank, world, port, grid_dims, Xl, q, allreduce):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    os.environ["B200_ALLREDUCE"] = allreduce
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    import oracle
    from common import CudaMem
    from quda_b200 import comm, dirac as DR, dslash as D, fields as F
    grid = comm.ProcessGrid(grid_dims, rank)
    Xg = [Xl[d] * grid_dims[d] for d in range(4)]
    kappa = 0.12195
    gauge = oracle.random_gauge(Xg, 8, seed=137)
    clover = oracle.random_clover(Xg, 8, seed=138)
    b = oracle.random_spinor(Xg, 8, seed=77, nparity=1)  # the even-parity source of the even-even Schur complement
    Vhl = F.volume_cb(Xl)

    def neighbours_gauge():
        out = []
        for d in range(4):
            c = list(grid.coords)
            c[d] = (c[d] - 1) % grid_dims[d]
            out.append(comm.local_slice(gauge, Xg, Xl, c, "gauge") if grid_dims[d] > 1 else None)
        return out

    ops, keep = {}, []
    for prec in (8, 4):
        ex = comm.HaloExchange(grid, Xl, prec, mode="p2p", dist=dist)
        cs = ex.comm_struct()
        gbuf, gmeta = F.gauge_to_native(comm.local_slice(gauge, Xg, Xl, grid.coords, "gauge"), Xl, prec, 12,
                                        ghost_from=neighbours_gauge())
        U = D.GaugeField(CudaMem.put(gbuf), Xl, prec, 12, gmeta, t_boundary=-1,
                         first_time_slice=grid.first_time_slice(), last_time_slice=grid.last_time_slice())
        cbuf, cmeta = F.clover_to_native(comm.local_slice(clover, Xg, Xl, grid.coords, "clover"), Xl, prec, compressed=True)
        A = D.CloverField(CudaMem.put(cbuf), Xl, prec, cmeta, dynamic=True)
        ops[prec] = DR.Dirac("cloverpc", U, kappa, clover=A, comm=cs)
        keep += [ex, cs, U, A]
    bl = comm.local_slice(b, Xg, Xl, grid.coords, ("spinor1", 0))
    pb = F.spinor_bytes(Xl, 8)
    bdev = D.ColorSpinorField(CudaMem.put(F.spinor_to_native(bl, 8)), Xl, 8)
    xs = [D.ColorSpinorField(CudaMem.empty(pb), Xl, 8) for _ in OFFSETS]
    res = DR.invert_multishift_cg(ops[8], ops[4], xs, bdev, OFFSETS, tol=1e-10, maxiter=3000)
    torch.cuda.synchronize()
    local = [F.spinor_from_native(CudaMem.get(x.buf), Vhl, 8) for x in xs]
    blocks = [None] * world
    dist.all_gather_object(blocks, (grid.coords, local))
    clover_inv = oracle.clover_invert(clover)
    Vhg = F.volume_cb(Xg)
    true_res = []
    for j, sigma in enumerate(OFFSETS):
        xg = np.zeros_like(b, dtype=np.float64)
        for coords, blk in blocks:
            off = np.array([coords[d] * Xl[d] for d in range(4)])
            xg[F.cb_index(F.cb_coords(Xl, 0) + off, Xg)] = blk[j]
        assert xg.shape[0] == Vhg
        m = lambda v, d: oracle.clover_matpc(gauge, clover, clover_inv, v, Xg, kappa, 0, d)  # noqa: E731
        r = m(m(xg, 0), 1) + sigma * xg - b
        true_res.append(float(np.linalg.norm(r.ravel()) / np.linalg.norm(b.ravel())))
    timed_out = any(e.timed_out() for e in keep if hasattr(e, "timed_out"))
    q.put((rank, res.iter, list(res.iter_offset[:len(OFFSETS)]), list(res.refine_iter[:len(OFFSETS)]), res.reliable_updates,
           list(res.true_res_offset[:len(OFFSETS)]), true_res, timed_out))
    dist.barrier()
    dist.destroy_process_group()
