#!/usr/bin/env python
"""Time gauge smearing on one GPU at 32^4 (--dim), fp64 and fp32, for every kind in 4-d and in 3-d (t ignored).  One
JSON line per (kind, dirs, precision): step_us is the device time of one call of one step out of place, from
torch.profiler over --reps calls: its kernels (gauge_stout_kernel or gauge_smear_level_kernel; HYP runs one per level)
plus, in 3-d, the device-to-device copy of the ignored direction (copy_us on its own); GB/s over the byte model below and
the fraction of 3.35 TB/s (the H100 SXM data-sheet HBM3 bandwidth).  The card's name and power limit are read in the same
run.

Byte model (prec = 8 or 4 bytes, V sites, d smeared directions, one link 18 prec; the neighbour links of the staples come
from cache, as for the gauge force and the flow):
  APE, stout, over-improved stout   per smeared link: read U, write U'                               2 d
  HYP level 1                       read U, write its d - 1 decorated links                          d d
  HYP level 2 (4-d)                 read U and its 3 level-1 links, write its 3 level-2 links        7 d
  HYP last level                    read U and its d - 1 decorated links, write U'                   (d + 1) d
  3-d: the copy of the ignored direction, read and write                                             2
per site and step, in links of 18 prec.

  python tools/bench_smear.py [--dim 32 32 32 32] [--reps 10] [--warmup 2]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

HBM = 3.35e12
COEFFS = {"ape": {"alpha": 0.6}, "stout": {"rho": 0.1}, "ovrimp_stout": {"rho": 0.06, "epsilon": -0.25},
          "hyp": {"alpha1": 0.75, "alpha2": 0.6, "alpha3": 0.3}}


def links_per_site(kind, d):
    copy = 2 if d == 3 else 0
    if kind != "hyp":
        return 2 * d + copy
    return d * d + (7 * d if d == 4 else 0) + (d + 1) * d + copy


def _device_us(fn, reps):
    """(device time of the smearing kernels, of the device-to-device copies, kernels launched) per call, from
    torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type.name == "CUDA"]
    kern = [e for e in ev if "gauge_stout_kernel" in e.name or "gauge_smear_level_kernel" in e.name]
    copy = [e for e in ev if "Memcpy" in e.name and "DtoD" in e.name]
    return sum(e.device_time for e in kern) / reps, sum(e.device_time for e in copy) / reps, len(kern) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dim", type=int, nargs=4, default=[32, 32, 32, 32])
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import torch

    from quda_b200 import gauge as GP
    from solver_bench import card
    assert torch.cuda.is_available(), "bench_smear.py measures on a CUDA device"
    info = card()
    X = a.dim
    V = X[0] * X[1] * X[2] * X[3]
    torch.manual_seed(1)
    g = torch.linalg.qr(torch.randn((4, V, 3, 3), dtype=torch.complex128, device="cuda"))[0]
    for prec in (8, 4):
        gauge = torch.view_as_real(g).to(torch.float64 if prec == 8 else torch.float32).contiguous()
        out = torch.empty_like(gauge)
        for kind in sorted(COEFFS):
            for ign in (4, 3):
                d = 4 if ign == 4 else 3

                def step():
                    GP.gauge_smear(out, gauge, kind, 1, X=X, dir_ignore=ign, **COEFFS[kind])

                for _ in range(a.warmup):
                    step()
                torch.cuda.synchronize()
                kus, cus, launches = _device_us(step, a.reps)
                us = kus + cus
                b = links_per_site(kind, d) * 18 * prec * V
                print(json.dumps(dict(kind=kind, dirs=d, dim=X, prec=prec, launches_per_step=launches, step_us=round(us, 1),
                                      copy_us=round(cus, 1),
                                      step_bytes=b, step_gbs=round(b / us / 1e3, 1),
                                      step_hbm_fraction=round(b / us / 1e-6 / HBM, 3), card=info)), flush=True)
    del out, gauge


if __name__ == "__main__":
    main()
