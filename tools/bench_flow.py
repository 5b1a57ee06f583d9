#!/usr/bin/env python
"""Time the gradient flow and the gauge observables on one GPU at 32^4 (--dim), fp64 and fp32, Wilson and Symanzik.  One
JSON line per (action, precision): stage_us is the device time of one RK3 stage kernel (gauge_flow_kernel) and step_us of
one step (three stages), obs_us of gauge_obs_kernel, all from torch.profiler over --reps calls; GB/s over the byte model
below and the fraction of 3.35 TB/s (the H100 SXM data-sheet HBM3 bandwidth); flow_s is the wall time of
gradient_flow to t = 1 at epsilon = 0.01 with a measurement every 10 steps (host clock around the call, after a
synchronise; it includes the stream-ordered scratch allocations and the synchronising observables).  The card's name and
power limit are read in the same run.

Byte model (prec = 8 or 4 bytes, V sites; the neighbour links of the staples and leaves come from cache, as for the gauge
force):
  RK3 step        each of the three stages reads and writes the links, 3 2 4 18 V prec; the accumulator [V][4][10] is
                  written by stage 1, read and written by stage 2 and read by stage 3, 4 4 10 V prec (fp64: 4736 B per site)
  observables     links 4 18 V prec, density 8 V

  python tools/bench_flow.py [--dim 32 32 32 32] [--reps 10] [--warmup 2]"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

HBM = 3.35e12


def step_bytes(V, p):
    return (3 * 2 * 4 * 18 + 4 * 4 * 10) * V * p


def obs_bytes(V, p):
    return 4 * 18 * V * p + 8 * V


def _kernel_us(fn, reps, name):
    """device time of the kernels named `name` per call, from torch.profiler, and how many ran per call"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type.name == "CUDA" and name in e.name]
    return sum(e.device_time for e in ev) / reps, len(ev) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dim", type=int, nargs=4, default=[32, 32, 32, 32])
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import torch

    from quda_b200 import gauge as GP
    from solver_bench import card
    assert torch.cuda.is_available(), "bench_flow.py measures on a CUDA device"
    info = card()
    X = a.dim
    V = X[0] * X[1] * X[2] * X[3]
    torch.manual_seed(1)
    g = torch.linalg.qr(torch.randn((4, V, 3, 3), dtype=torch.complex128, device="cuda"))[0]
    for action in sorted(GP.FLOW_ACTIONS):
        paths, coeffs = GP.FLOW_ACTIONS[action]
        for prec in (8, 4):
            gauge = torch.view_as_real(g).to(torch.float64 if prec == 8 else torch.float32).contiguous()
            out = torch.empty_like(gauge)
            dens = torch.empty(V, dtype=torch.float64, device="cuda")

            def step():
                GP.gauge_flow(out, gauge, 0.01, 1, paths, coeffs, X=X)

            def obs():
                GP.gauge_observables(gauge, X=X, density=dens)

            for _ in range(a.warmup):
                step()
                obs()
            torch.cuda.synchronize()
            step_us, stages = _kernel_us(step, a.reps, "gauge_flow_kernel")
            obs_us, _ = _kernel_us(obs, a.reps, "gauge_obs_kernel")
            GP.gradient_flow(gauge, 0.01, 10, X=X, action=action, meas_interval=10)  # warm the measured path
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            _, rows = GP.gradient_flow(gauge, 0.01, 100, X=X, action=action, meas_interval=10)
            torch.cuda.synchronize()
            flow_s = time.perf_counter() - t0
            sb, ob = step_bytes(V, prec), obs_bytes(V, prec)
            print(json.dumps(dict(action=action, dim=X, prec=prec, paths=len(coeffs), stages_per_step=stages,
                                  stage_us=round(step_us / stages, 2), step_us=round(step_us, 2), step_bytes=sb,
                                  step_gbs=round(sb / step_us / 1e3, 1), step_hbm_fraction=round(sb / step_us / 1e-6 / HBM, 3),
                                  obs_us=round(obs_us, 2), obs_bytes=ob, obs_gbs=round(ob / obs_us / 1e3, 1),
                                  obs_hbm_fraction=round(ob / obs_us / 1e-6 / HBM, 3), flow_to_t1_s=round(flow_s, 3),
                                  t2E_at_t1=rows[-1][0] ** 2 * rows[-1][2][0], card=info)), flush=True)


if __name__ == "__main__":
    main()
