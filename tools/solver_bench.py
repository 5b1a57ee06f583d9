"""Set-up shared by the solver benchmarks (tools/bench_bicgstab.py, tools/bench_multishift.py): one process per GPU from
torchrun's environment, the global lattice split over the ranks, the Wilson-clover even-even preconditioned operator in
double (recon 18) and single (recon 12) precision, and the alternating CUDA-event timing loop."""
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


def setup(global_dim, kappa):
    """Join the ranks (none with one process), split the global lattice and build the clover-PC operators on this rank's
    block on the current stream.  Returns (rank, world, dist, dims, X, ops) with ops[8] double, ops[4] single precision;
    dist is None for one process."""
    import torch
    from quda_b200 import comm, dirac as DR, dslash as D, fields as F
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    assert torch.cuda.is_available(), f"{os.path.basename(sys.argv[0])} needs a CUDA device (no CPU fallback)"
    torch.cuda.set_device(local_rank)
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    dims = comm.ProcessGrid.default_dims(world)
    grid = comm.ProcessGrid(dims, rank) if world > 1 else None
    Xg = global_dim
    X = [Xg[d] // dims[d] for d in range(4)]
    assert all(X[d] * dims[d] == Xg[d] and X[d] % 2 == 0 for d in range(4)), f"global lattice {Xg} does not split over {dims}"
    torch.manual_seed(4321 + rank)
    u = bench.random_su3_device(X)
    faces = bench.boundary_links_from_neighbours(u, X, grid)
    ops = {}
    stream = torch.cuda.current_stream().cuda_stream
    for prec, recon in ((8, 18), (4, 12)):
        gbuf, gmeta = F.gauge_to_native_torch(u, X, prec, recon, ghost_faces=faces)
        U = D.GaugeField(gbuf, X, prec, recon, gmeta, anisotropy=1.0, t_boundary=-1,
                         first_time_slice=grid.first_time_slice() if grid else True,
                         last_time_slice=grid.last_time_slice() if grid else True)
        A = bench.device_clover(X, prec)
        ex = cs = None
        if world > 1:
            ex = comm.HaloExchange(grid, X, prec, mode="p2p", dist=dist)
            cs = ex.comm_struct()
        ops[prec] = DR.Dirac("cloverpc", U, kappa, clover=A, comm=cs, stream=stream)
        ops[prec]._keep = ex  # the comm block points into the exchange's buffers
    return rank, world, dist, dims, X, ops


def timed_runs(modes, solve, reps, dist):
    """One warm-up solve(mode) per mode, then `reps` rounds that time every mode in turn with CUDA events.  Yields
    (mode, seconds, solve's result) after each timed solve."""
    import torch
    for m in modes:
        solve(m)  # warm-up: first-use allocations, clocks
    for _ in range(reps):
        for m in modes:
            if dist is not None:
                dist.barrier()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            res = solve(m)
            e1.record()
            torch.cuda.synchronize()
            yield m, e0.elapsed_time(e1) * 1e-3, res


def max_over_ranks(dist, *values):
    """the largest of each value over the ranks (the values themselves with one process)"""
    if dist is None:
        return values
    import torch
    t = torch.tensor(values, device="cuda", dtype=torch.float64)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return [float(v) for v in t]
