"""Multi-rank workers: every rank owns one block of a global lattice and exchanges halos with its neighbours, and every
result is checked against the oracle on the GLOBAL lattice.  `worker` applies x + a D in (mode "host": gloo + host twin,
CPU tier; "p2p"/"nccl": one GPU per rank, libquda_b200.so, NVLink peer writes / NCCL send-recv, GPU tier).
`solver_worker` runs CG, BiCGStab or multi-shift CG through the C++ operator / solver layer, one GPU per rank.
`run_ranks` spawns the ranks of either and collects one result dict per rank."""
import os
import socket
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def run_ranks(target, world, args, timeout):
    """Run target(rank, world, port, q, *args) in `world` spawned processes and return the result every rank puts on q.
    Each rank must exit cleanly, and none outlives this call: a hung rank would hold its GPU and starve every later test."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=target, args=(r, world, port, q, *args)) for r in range(world)]
    try:
        for p in procs:
            p.start()
        res = [q.get(timeout=timeout) for _ in procs]
        for p in procs:
            p.join(timeout=120)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(timeout=30)
    return res


def _join(rank, world, port, backend):
    """Put the repository on the path and join the process group (nccl: this rank's GPU is cuda:rank)."""
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    import torch
    import torch.distributed as dist
    if backend == "nccl":
        torch.cuda.set_device(rank)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    else:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    return dist


def _leave(dist, q, result):
    q.put(result)
    dist.barrier()
    dist.destroy_process_group()


class Block:
    """This rank's block of a global lattice: native local fields cut from global oracle-order ones (every rank builds the
    same global fields from the same seeds), and the gather of every rank's block back onto the global lattice."""

    def __init__(self, grid, Xl, mem):
        self.grid, self.Xl, self.mem = grid, [int(v) for v in Xl], mem
        self.Xg = [self.Xl[d] * grid.dims[d] for d in range(4)]

    def gauge_field(self, gauge, prec, recon):
        """the local links, with the backward neighbours' links in the pad"""
        from quda_b200 import comm, dslash as D, fields as F
        g = self.grid
        ghost_from = []
        for d in range(4):
            c = list(g.coords)
            c[d] = (c[d] - 1) % g.dims[d]
            ghost_from.append(comm.local_slice(gauge, self.Xg, self.Xl, c, "gauge") if g.dims[d] > 1 else None)
        gbuf, gmeta = F.gauge_to_native(comm.local_slice(gauge, self.Xg, self.Xl, g.coords, "gauge"), self.Xl, prec, recon,
                                        ghost_from=ghost_from)
        return D.GaugeField(self.mem.put(gbuf), self.Xl, prec, recon, gmeta, t_boundary=-1,
                            first_time_slice=g.first_time_slice(), last_time_slice=g.last_time_slice())

    def clover_field(self, clover, prec):
        """the local clover term, compressed, with its inverse computed on the fly"""
        from quda_b200 import comm, dslash as D, fields as F
        cbuf, cmeta = F.clover_to_native(comm.local_slice(clover, self.Xg, self.Xl, self.grid.coords, "clover"), self.Xl,
                                         prec, compressed=True)
        return D.CloverField(self.mem.put(cbuf), self.Xl, prec, cmeta, dynamic=True)

    def spinor_field(self, v, prec, parity=None):
        """the local sites of a single-parity global spinor of the given parity, or of a two-parity one ([even | odd])"""
        from quda_b200 import comm, dslash as D, fields as F
        if parity is not None:
            buf = F.spinor_to_native(comm.local_slice(v, self.Xg, self.Xl, self.grid.coords, ("spinor1", parity)), prec)
            return D.ColorSpinorField(self.mem.put(buf), self.Xl, prec)
        local, Vhl = comm.local_slice(v, self.Xg, self.Xl, self.grid.coords, "spinor2"), F.volume_cb(self.Xl)
        buf = np.concatenate([F.spinor_to_native(local[p * Vhl:(p + 1) * Vhl], prec) for p in range(2)])
        return D.ColorSpinorField(self.mem.put(buf), self.Xl, prec, 2)

    def empty(self, prec, nparity=1):
        from quda_b200 import dslash as D, fields as F
        return D.ColorSpinorField(self.mem.empty(nparity * F.spinor_bytes(self.Xl, prec)), self.Xl, prec, nparity)

    def to_host(self, field):
        """a local field in oracle order"""
        from quda_b200 import fields as F
        self.mem.sync()
        raw, pb = self.mem.get(field.buf), field.parity_bytes
        return np.concatenate([F.spinor_from_native(raw[p * pb:(p + 1) * pb], F.volume_cb(self.Xl), field.prec)
                               for p in range(field.n_parity)])

    def gather(self, dist, fields, parity=0):
        """every rank's block of each local field onto the global lattice, on the host in fp64; a single-parity field holds
        the sites of `parity`"""
        from quda_b200 import fields as F
        Vhl, Vhg = F.volume_cb(self.Xl), F.volume_cb(self.Xg)
        blocks = [None] * self.grid.size
        dist.all_gather_object(blocks, (self.grid.coords, [self.to_host(f) for f in fields]))
        out = []
        for j, f in enumerate(fields):
            parities = range(2) if f.n_parity == 2 else [parity]
            g = np.zeros((len(parities) * Vhg,) + blocks[0][1][j].shape[1:], dtype=np.float64)
            for coords, local in blocks:
                off = np.array([coords[d] * self.Xl[d] for d in range(4)])
                for i, p in enumerate(parities):
                    g[i * Vhg + F.cb_index(F.cb_coords(self.Xl, p) + off, self.Xg)] = local[j][i * Vhl:(i + 1) * Vhl]
            out.append(g)
        return out


def worker(rank, world, port, q, grid_dims, Xl, prec, recon, mode="host", reps=3, n_src=1):
    """x + a D in for the Wilson Dslash on this rank's block; reports the deviation from the global oracle."""
    os.environ["OMP_NUM_THREADS"] = "2"
    fused = mode == "p2p-fused"  # the C++ operator layer's schedule: pack + interior + boundary as ONE launch per Dslash
    if fused:
        mode = "p2p"
    dist = _join(rank, world, port, "gloo" if mode == "host" else "nccl")
    import oracle
    import ops
    from common import CudaMem, HostMem, twin_backend
    from quda_b200 import comm
    be = twin_backend() if mode == "host" else None
    grid = comm.ProcessGrid(grid_dims, rank)
    blk = Block(grid, Xl, HostMem if mode == "host" else CudaMem)
    Xg = blk.Xg
    hp = 8 if prec == 8 else 4
    gauge = oracle.random_gauge(Xg, hp, seed=137)          # same global field on every rank (same seed)
    parity, dagger, kappa = 1, 0, 0.12195
    s = oracle.random_spinor(Xg, hp, seed=5)
    xs = oracle.random_spinor(Xg, hp, seed=6)
    ref = ops.xpay(xs, -kappa, oracle.wil_dslash(gauge, s, Xg, parity, dagger))
    U = blk.gauge_field(gauge, prec, recon)
    din, dx, out = blk.spinor_field(s, prec, 1 - parity), blk.spinor_field(xs, prec, parity), blk.empty(prec)
    if n_src > 1:
        # a multi-RHS batch: ONE batched exchange (one pack launch / one message per face for all sources), then every
        # source's Dslash on its own ghost slab; source i is s rolled by i sites so that the sources differ
        ex = comm.HaloExchange(grid, Xl, prec, mode=mode, backend=be, dist=dist, n_src=n_src)
        srcs = [np.roll(s, i, axis=0) for i in range(n_src)]
        dins = [blk.spinor_field(v, prec, 1 - parity) for v in srcs]
        outs = [blk.empty(prec) for _ in range(n_src)]
        for _ in range(reps):
            comm.apply_wilson_distributed(ex, outs, dins, U, -kappa, [dx] * n_src, parity, dagger)
        comm.apply_wilson_distributed(ex, out, din, U, -kappa, dx, parity, dagger)  # a single exchange on the same buffers
        dev = 0.0
        for i in range(n_src + 1):
            v, o = (srcs[i], outs[i]) if i < n_src else (s, out)
            r = ops.xpay(xs, -kappa, oracle.wil_dslash(gauge, v, Xg, parity, dagger))
            dev = max(dev, oracle.compare_spinor(comm.local_slice(r, Xg, Xl, grid.coords, ("spinor1", parity)), blk.to_host(o))[1])
    else:
        ex = comm.HaloExchange(grid, Xl, prec, mode=mode, backend=be, dist=dist)
        if fused:
            from quda_b200 import dirac as DR
            op = DR.Dirac("wilson", U, 0.0, comm=ex.comm_struct())
            for _ in range(reps):
                op.DslashXpay(out, din, parity, dx, -kappa, dagger=bool(dagger))
        else:
            for _ in range(reps):  # repeated applications exercise the double-buffered ghost zones
                comm.apply_wilson_distributed(ex, out, din, U, -kappa, dx, parity, dagger)
        want = comm.local_slice(ref, Xg, Xl, grid.coords, ("spinor1", parity))
        dev = oracle.compare_spinor(want, blk.to_host(out))[1]
    _leave(dist, q, {"rank": rank, "dev": dev, "timed_out": ex.timed_out()})


def solver_worker(rank, world, port, q, grid_dims, Xl, solver, kind="cloverpc", mixed=True, allreduce=None):
    """One solve to 1e-10 through the C++ operator / solver layer: every Dslash inside the solver exchanges its halo over
    NVLink, and the scalars are all-reduced in the reduction kernels (NVLink mailboxes, B200_ALLREDUCE=nvlink) or through
    the host callback (B200_ALLREDUCE=callback); None keeps the library's default.  CG solves the normal equations and
    BiCGStab M_pc itself, both through prepare / reconstruct, and the gathered solution must satisfy M x = b with the
    oracle's full operator (invert_test's criterion).  Multi-shift CG solves (M_pc^dag M_pc + sigma_j) x_j = b for the
    even-even clover-PC operator, and every gathered x_j is checked with the oracle's M_pc."""
    if allreduce is not None:
        os.environ["B200_ALLREDUCE"] = allreduce
    dist = _join(rank, world, port, "nccl")
    import oracle
    from common import CudaMem
    from quda_b200 import comm, dirac as DR
    from solvers import KAPPA as kappa, OFFSETS, solve_prepared
    grid = comm.ProcessGrid(grid_dims, rank)
    blk = Block(grid, Xl, CudaMem)
    Xg = blk.Xg
    gauge = oracle.random_gauge(Xg, 8, seed=137)
    clover = oracle.random_clover(Xg, 8, seed=138) if "clover" in kind else None
    b = oracle.random_spinor(Xg, 8, seed=77, nparity=1 if solver == "multishift" else 2)
    ops, exs = {}, []
    for prec in ((8, 4) if mixed else (8,)):
        ex = comm.HaloExchange(grid, Xl, prec, mode="p2p", dist=dist)
        cs = ex.comm_struct()
        U = blk.gauge_field(gauge, prec, 12)
        A = blk.clover_field(clover, prec) if clover is not None else None
        ops[prec] = DR.Dirac(kind, U, kappa, clover=A, comm=cs)
        exs.append(ex)
    out = {"rank": rank}
    if solver == "multishift":
        bdev = blk.spinor_field(b, 8, parity=0)  # the even-parity source of the even-even Schur complement
        xs = [blk.empty(8) for _ in OFFSETS]
        res = DR.invert_multishift_cg(ops[8], ops[4], xs, bdev, OFFSETS, tol=1e-10, maxiter=3000)
        clover_inv = oracle.clover_invert(clover)
        m = lambda v, d: oracle.clover_matpc(gauge, clover, clover_inv, v, Xg, kappa, 0, d)  # noqa: E731
        n = len(OFFSETS)
        out.update(iter_offset=list(res.iter_offset[:n]), refine_iter=list(res.refine_iter[:n]),
                   true_res_offset=list(res.true_res_offset[:n]),
                   host_true_res=[float(np.linalg.norm((m(m(x, 0), 1) + sigma * x - b).ravel()) / np.linalg.norm(b.ravel()))
                                  for sigma, x in zip(OFFSETS, blk.gather(dist, xs, parity=0))])
    else:
        bdev, xdev = blk.spinor_field(b, 8), blk.empty(8, 2)
        res = solve_prepared(ops[8], ops.get(4), solver, xdev, bdev, maxiter=3000)
        (x,) = blk.gather(dist, [xdev])
        if clover is None:
            Mx = oracle.wil_mat(gauge, x, Xg, kappa, 0)
        else:
            Mx = oracle.clover_mat(gauge, clover, x, Xg, kappa, 0)
        out.update(true_res=res.true_res, host_true_res=float(np.linalg.norm(Mx.ravel() - b.ravel()) / np.linalg.norm(b.ravel())))
    out.update(iter=res.iter, reliable_updates=res.reliable_updates, timed_out=any(e.timed_out() for e in exs))
    _leave(dist, q, out)
