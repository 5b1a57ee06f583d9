#!/usr/bin/env python
"""Time the gauge half of an HMC step on one GPU at 32^4 (--dim), fp64 and fp32.  One JSON line per call: us is the device
time of the library's kernels per call (torch.profiler over --reps calls), us_call the whole call (CUDA events over --reps
calls after --warmup calls; for the two sums it includes the stream-ordered allocation of their partial sums and the
synchronisation); bytes from the model below, GB/s and the fraction of 3.35 TB/s (the H100 SXM data-sheet HBM3 bandwidth)
over us.  Then, in fp64, the wall time of one two-flavour clover HMC trajectory at 16^3x32 (--traj-dim, --steps leapfrog
steps) split into solves, fermion force, gauge force, link updates and clover rebuilds (load_gauge + compute_clover_field).
The card's name and power limit are read in the same run.

Byte model (prec = 8 or 4 bytes, V sites; every field read or written once):
  gauge_force     links 4 18 V prec; mom read and written 2 4 10 V prec (the paths reread links from cache)
  update_gauge    links read and written 2 4 18 V prec; mom 4 10 V prec
  mom_action      mom 4 10 V prec
  plaquette       links 4 18 V prec

  python tools/bench_gauge.py [--dim 32 32 32 32] [--reps 20] [--warmup 3] [--traj-dim 16 16 16 32] [--steps 10]"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM = 3.35e12
BYTES = {
    "gauge_force": lambda V, p: (4 * 18 + 2 * 4 * 10) * V * p,
    "update_gauge": lambda V, p: (2 * 4 * 18 + 4 * 10) * V * p,
    "mom_action": lambda V, p: 4 * 10 * V * p,
    "plaquette": lambda V, p: 4 * 18 * V * p,
}


def _time(fn, reps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        fn()
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) * 1e3 / reps


def _kernel_us(fn, reps):
    """device time of the library's kernels per call, from torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    return sum(e.device_time for e in prof.events() if e.device_type.name == "CUDA" and "b200::" in e.name) / reps


def kernels(a, info):
    import torch

    import gauge_cases as GC
    from quda_b200 import gauge as GP
    X = a.dim
    V = X[0] * X[1] * X[2] * X[3]
    g = torch.linalg.qr(torch.randn((4, V, 3, 3), dtype=torch.complex128, device="cuda"))[0]
    for prec in (8, 4):
        dt = torch.float64 if prec == 8 else torch.float32
        gauge = torch.view_as_real(g).to(dt).contiguous()
        out = torch.empty_like(gauge)
        mom = (0.1 * torch.randn((V, 4, 10), dtype=torch.float64, device="cuda")).to(dt)
        rows = []
        for name in ("plaq", "plaq+rect"):
            p, c = GC.path_set(name)
            rows.append((f"gauge_force[{len(c)} paths]", "gauge_force",
                         lambda p=p, c=c: GP.gauge_force(mom, gauge, p, c, 1e-6, X=X)))
        rows.append(("update_gauge[exact]", "update_gauge", lambda: GP.update_gauge_field(gauge, mom, 0.01, X=X, out=out)))
        rows.append(("update_gauge[order 8]", "update_gauge",
                     lambda: GP.update_gauge_field(gauge, mom, 0.01, exact=False, X=X, out=out)))
        rows.append(("mom_action", "mom_action", lambda: GP.mom_action(mom, X=X)))
        rows.append(("plaquette", "plaquette", lambda: GP.plaquette(gauge, X=X)))
        for label, model, fn in rows:
            us_call = _time(fn, a.reps, a.warmup)
            us = _kernel_us(fn, a.reps)
            nbytes = BYTES[model](V, prec)
            print(json.dumps(dict(call=label, dim=X, prec=prec, us=round(us, 2), us_call=round(us_call, 2), bytes=nbytes,
                                  gbs=round(nbytes / us / 1e3, 1),
                                  hbm_fraction=round(nbytes / us / 1e-6 / HBM, 3), card=info)), flush=True)


def trajectory(a, info):
    """one two-flavour clover HMC trajectory, leapfrog, tau = 1, fp64, asymmetric even-even clover-PC operator"""
    import numpy as np
    import torch

    import gauge_cases as GC
    from common import CudaMem, Problem
    from quda_b200 import dirac as DR
    from quda_b200 import dslash as D
    from quda_b200 import gauge as GP
    kappa, csw, beta, tau = 0.12, 1.3, 5.5, 1.0
    X = a.traj_dim
    V = int(np.prod(X))
    P = Problem(X, 8, 18, CudaMem)
    U = torch.from_numpy(GC.antiperiodic(GC.near_identity_links(X, 1, 0.1), X)).cuda()
    mom = torch.from_numpy(GC.random_mom(V, 2)).cuda()
    paths, coeffs = GC.path_set("plaq")
    t = dict(solves=0.0, fermion_force=0.0, gauge_force=0.0, updates=0.0, clover_rebuilds=0.0)

    def timed(key, fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        t[key] += time.perf_counter() - t0
        return r

    def operator():
        def build():
            Un = D.load_gauge(U, X, 8, 18, t_boundary=-1)
            A, Ainv, _ = D.compute_clover_field(U, X, 8, kappa, csw)
            return DR.Dirac("cloverpc", Un, kappa, clover=A, clover_inv=Ainv, matpc_type=DR.MATPC_EVEN_EVEN_ASYMMETRIC)
        return timed("clover_rebuilds", build)

    op = operator()
    phi = P.empty(1)
    op.Mdag(phi, P.to_dev(np.random.default_rng(3).normal(size=(V // 2, 4, 3, 2)) * np.sqrt(0.5)))
    iters = []
    for k in t:  # the first operator (and its warm-up) is not part of the trajectory
        t[k] = 0.0

    def kick(eps):
        timed("gauge_force", lambda: GP.gauge_force(mom, U, paths, coeffs, eps * beta / 3, X=X))
        x = P.empty(1)
        p = timed("solves", lambda: DR.invert_multishift_cg(op, None, [x], phi, [0.0], tol=1e-10))
        iters.append(p.iter)
        timed("fermion_force", lambda: DR.compute_clover_force(mom, eps, [x], [1.0], kappa, csw, 2, U, op))

    n = a.steps
    dt = tau / n
    torch.cuda.synchronize()
    t_all = time.perf_counter()
    kick(0.5 * dt)
    for i in range(n):
        timed("updates", lambda: GP.update_gauge_field(U, mom, dt, X=X, out=U))
        op = operator()
        kick(dt if i < n - 1 else 0.5 * dt)
    torch.cuda.synchronize()
    total = time.perf_counter() - t_all
    print(json.dumps(dict(trajectory="two-flavour clover HMC, leapfrog", dim=X, prec=8, steps=n, total_s=round(total, 3),
                          **{k + "_s": round(v, 4) for k, v in t.items()}, cg_iters=iters, card=info)), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dim", type=int, nargs=4, default=[32, 32, 32, 32])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--traj-dim", type=int, nargs=4, default=[16, 16, 16, 32])
    ap.add_argument("--steps", type=int, default=10)
    a = ap.parse_args()
    import torch

    from solver_bench import card
    assert torch.cuda.is_available(), "bench_gauge.py measures on a CUDA device"
    info = card()
    kernels(a, info)
    trajectory(a, info)


if __name__ == "__main__":
    main()
