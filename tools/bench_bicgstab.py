#!/usr/bin/env python
"""Time CG on the normal equations against BiCGStab on M_pc for `bench.py --op cg`'s system: Wilson-clover, symmetric
even-even preconditioning, double precision with a single-precision sloppy operator and reliable updates, global lattice
--global-dim (default 48^3 x 96) split over the ranks.

  python tools/bench_bicgstab.py [--global-dim X Y Z T] [--tol 1e-10] [--reps 1]
  torchrun --nproc-per-node N tools/bench_bicgstab.py ...

Each solver gets one warm-up solve, then the two are timed alternately with CUDA events (prepare + solve + reconstruct).
One JSON line per solver: iterations, M applications (two per iteration for both, plus the residual recomputations),
reliable updates (BiCGStab: including restarts), time to solution, GFLOP/s with the library's accounting, the full-system
true residual from the unpreconditioned fp64 operator, and the card and its power limit."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (field helpers: random SU(3) links, ghost links, device clover)


def card():
    import torch
    out = {"name": torch.cuda.get_device_name(), "power_limit_w": None}
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                                     str(torch.cuda.current_device())], timeout=10).decode().strip()
        out["power_limit_w"] = float(q)
    except Exception as e:  # noqa: BLE001
        out["power_limit_w"] = f"unavailable ({e.__class__.__name__})"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--global-dim", type=int, nargs=4, default=[48, 48, 48, 96])
    ap.add_argument("--tol", type=float, default=1e-10)
    ap.add_argument("--kappa", type=float, default=0.12195)
    ap.add_argument("--reps", type=int, default=1, help="timed solves per solver (alternating)")
    a = ap.parse_args()

    import torch
    from quda_b200 import comm, dirac as DR, dslash as D, fields as F
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    assert torch.cuda.is_available(), "bench_bicgstab.py needs a CUDA device (no CPU fallback)"
    torch.cuda.set_device(local_rank)
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    dims = comm.ProcessGrid.default_dims(world)
    grid = comm.ProcessGrid(dims, rank) if world > 1 else None
    Xg = a.global_dim
    X = [Xg[d] // dims[d] for d in range(4)]
    assert all(X[d] * dims[d] == Xg[d] and X[d] % 2 == 0 for d in range(4)), f"global lattice {Xg} does not split over {dims}"
    torch.manual_seed(4321 + rank)
    u = bench.random_su3_device(X)
    faces = bench.boundary_links_from_neighbours(u, X, grid)
    ops, keep = {}, []
    stream = torch.cuda.current_stream().cuda_stream
    for prec, recon in ((8, 18), (4, 12)):
        gbuf, gmeta = F.gauge_to_native_torch(u, X, prec, recon, ghost_faces=faces)
        U = D.GaugeField(gbuf, X, prec, recon, gmeta, anisotropy=1.0, t_boundary=-1,
                         first_time_slice=grid.first_time_slice() if grid else True,
                         last_time_slice=grid.last_time_slice() if grid else True)
        A = bench.device_clover(X, prec)
        cs = None
        if world > 1:
            ex = comm.HaloExchange(grid, X, prec, mode="p2p", dist=dist)
            cs = ex.comm_struct()
            keep += [ex, cs]
        ops[prec] = DR.Dirac("cloverpc", U, a.kappa, clover=A, comm=cs, stream=stream)
        keep += [U, A]
    del u
    pc = ops[8]
    pb = F.spinor_bytes(X, 8)
    g = torch.Generator(device="cuda").manual_seed(99 + rank)
    b = torch.rand(2 * pb // 8, dtype=torch.float64, device="cuda", generator=g).view(torch.uint8)
    bdev = D.ColorSpinorField(b, X, 8, 2)
    xdev = D.ColorSpinorField(torch.zeros(2 * pb, dtype=torch.uint8, device="cuda"), X, 8, 2)
    rhs = D.ColorSpinorField(torch.zeros(pb, dtype=torch.uint8, device="cuda"), X, 8)
    full = DR.Dirac("clover", ops[8].U, a.kappa, clover=ops[8].clover, comm=ops[8].comm, stream=stream)
    Mx = D.ColorSpinorField(torch.zeros(2 * pb, dtype=torch.uint8, device="cuda"), X, 8, 2)

    def solve(which):
        xdev.buf.zero_()
        src_p, sol_p = pc.prepare(xdev, bdev)
        src = D.ColorSpinorField(xdev.buf[src_p * pb:(src_p + 1) * pb], X, 8)
        sol = D.ColorSpinorField(xdev.buf[sol_p * pb:(sol_p + 1) * pb], X, 8)
        if which == "cg":
            pc.Mdag(rhs, src)  # normal equations: M^dag M x = M^dag src
        else:
            rhs.buf.copy_(src.buf)
        sol.buf.zero_()
        fn = DR.invert_cg if which == "cg" else DR.invert_bicgstab
        res = fn(pc, ops[4], sol, rhs, tol=a.tol, maxiter=20000)
        pc.reconstruct(xdev, bdev)
        return res

    def true_residual():
        full.M(Mx, xdev)
        torch.cuda.synchronize()
        d2 = (Mx.buf.view(torch.float64) - bdev.buf.view(torch.float64)).pow(2).sum()
        nrm = torch.stack([d2, bdev.buf.view(torch.float64).pow(2).sum()])
        if world > 1:
            dist.all_reduce(nrm)
        return float((nrm[0] / nrm[1]).sqrt())

    solvers = ("cg", "bicgstab")
    for s in solvers:
        solve(s)  # warm-up: first-use allocations, clocks
    runs = {s: [] for s in solvers}
    for _ in range(a.reps):
        for s in solvers:
            if world > 1:
                dist.barrier()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            res = solve(s)
            e1.record()
            torch.cuda.synchronize()
            secs = e0.elapsed_time(e1) * 1e-3
            runs[s].append((secs, res, true_residual()))
    info = card()
    for s in solvers:
        secs, res, tr = min(runs[s], key=lambda r: r[0])
        if world > 1:
            t = torch.tensor([secs, res.secs], device="cuda", dtype=torch.float64)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            secs, solver_secs = float(t[0]), float(t[1])
        else:
            solver_secs = res.secs
        # residual recomputations in the precise operator: the initial and final one and one per reliable update, each
        # M^dag M (2 M) for CG and M for BiCGStab; BiCGStab also applies M twice in the iteration queued behind the one
        # that converged (its BLAS kernels return at once)
        extra = 2 * (res.reliable_updates + 2) if s == "cg" else res.reliable_updates + 2 + 2
        out = {"solver": s, "system": "MdagM x = Mdag b (normal equations)" if s == "cg" else "M_pc x = b",
               "iterations": res.iter, "m_applications": 2 * res.iter + extra, "reliable_updates": res.reliable_updates, "time_to_solution_s": secs, "solver_secs": solver_secs,
               "gflops": res.gflops * res.secs / solver_secs * world, "true_res_full_system": tr,
               "solver_true_res": res.true_res, "host_syncs": res.host_syncs, "timed_solves": len(runs[s]),
               "global_dim": Xg, "grid": dims, "n_gpus": world, "tol": a.tol, "kappa": a.kappa,
               "precision": "double recon-18 / single recon-12 sloppy", "card": info["name"],
               "power_limit_w": info["power_limit_w"]}
        if rank == 0:
            print(json.dumps(out))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
