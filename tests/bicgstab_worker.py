"""Two-rank BiCGStab worker: every rank owns one block of a global lattice, the C++ solver layer exchanges every Dslash halo
over NVLink and all-reduces the complex scalars either in the reduction kernels (NVLink mailboxes, B200_ALLREDUCE=nvlink) or
through the host callback (B200_ALLREDUCE=callback).  The gathered solution is verified on the GLOBAL lattice with the
oracle's full operator."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def bicgstab_worker(rank, world, port, grid_dims, Xl, q, allreduce, kind="cloverpc", mixed=True):
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
    clover = oracle.random_clover(Xg, 8, seed=138) if "clover" in kind else None
    b = oracle.random_spinor(Xg, 8, seed=77, nparity=2)
    Vhl = F.volume_cb(Xl)

    def neighbours_gauge():
        out = []
        for d in range(4):
            c = list(grid.coords)
            c[d] = (c[d] - 1) % grid_dims[d]
            out.append(comm.local_slice(gauge, Xg, Xl, c, "gauge") if grid_dims[d] > 1 else None)
        return out

    ops, keep = {}, []
    for prec in ((8, 4) if mixed else (8,)):
        ex = comm.HaloExchange(grid, Xl, prec, mode="p2p", dist=dist)
        cs = ex.comm_struct()
        gbuf, gmeta = F.gauge_to_native(comm.local_slice(gauge, Xg, Xl, grid.coords, "gauge"), Xl, prec, 12,
                                        ghost_from=neighbours_gauge())
        U = D.GaugeField(CudaMem.put(gbuf), Xl, prec, 12, gmeta, t_boundary=-1,
                         first_time_slice=grid.first_time_slice(), last_time_slice=grid.last_time_slice())
        A = None
        if clover is not None:
            cbuf, cmeta = F.clover_to_native(comm.local_slice(clover, Xg, Xl, grid.coords, "clover"), Xl, prec, compressed=True)
            A = D.CloverField(CudaMem.put(cbuf), Xl, prec, cmeta, dynamic=True)
        ops[prec] = DR.Dirac(kind, U, kappa, clover=A, comm=cs)
        keep += [ex, cs, U, A]
    pc = ops[8]
    half = len(b) // 2
    bl = np.concatenate([comm.local_slice(b[p * half:(p + 1) * half], Xg, Xl, grid.coords, ("spinor1", p)) for p in range(2)])
    pb = F.spinor_bytes(Xl, 8)
    bdev = D.ColorSpinorField(CudaMem.put(np.concatenate([F.spinor_to_native(bl[p * Vhl:(p + 1) * Vhl], 8) for p in range(2)])), Xl, 8, 2)
    xdev = D.ColorSpinorField(CudaMem.empty(2 * pb), Xl, 8, 2)
    src_p, sol_p = pc.prepare(xdev, bdev)
    src = D.ColorSpinorField(CudaMem.empty(pb), Xl, 8)
    src.buf.copy_(xdev.buf[src_p * pb:(src_p + 1) * pb])
    sol = D.ColorSpinorField(xdev.buf[sol_p * pb:(sol_p + 1) * pb], Xl, 8)
    sol.buf.zero_()
    res = DR.invert_bicgstab(pc, ops.get(4), sol, src, tol=1e-10, maxiter=3000)
    pc.reconstruct(xdev, bdev)
    torch.cuda.synchronize()
    raw = CudaMem.get(xdev.buf)
    xl = np.concatenate([F.spinor_from_native(raw[p * pb:(p + 1) * pb], Vhl, 8) for p in range(2)])
    xg = np.zeros_like(b, dtype=np.float64)
    Vhg = F.volume_cb(Xg)
    blocks = [None] * world
    dist.all_gather_object(blocks, (grid.coords, xl))
    for coords, blk in blocks:
        off = np.array([coords[d] * Xl[d] for d in range(4)])
        for p in range(2):
            xg[p * Vhg + F.cb_index(F.cb_coords(Xl, p) + off, Xg)] = blk[p * Vhl:(p + 1) * Vhl]
    if clover is None:
        Mx = oracle.wil_mat(gauge, xg, Xg, kappa, 0)
    else:
        Mx = oracle.clover_mat(gauge, clover, xg, Xg, kappa, 0)
    true_res = float(np.linalg.norm(Mx.ravel() - b.ravel()) / np.linalg.norm(b.ravel()))
    timed_out = any(e.timed_out() for e in keep if hasattr(e, "timed_out"))
    q.put((rank, res.iter, res.reliable_updates, res.true_res, true_res, timed_out))
    dist.barrier()
    dist.destroy_process_group()
