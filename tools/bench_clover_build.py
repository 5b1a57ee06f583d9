#!/usr/bin/env python
"""Time the clover construction on one GPU: b200_compute_clover (links -> packed A) and b200_clover_invert_packed (A ->
A^-1 and tr log A) at 32^4 (--dim), fp64 and fp32, with CUDA events over --reps calls after --warmup calls.  One JSON line
per (call, precision) with microseconds per call, GB/s and GFLOP/s over the models below, and the card's name and power
limit read in the same run.  This is a set-up path: there is no speed target.

Byte model (compulsory traffic, prec = 8 or 4 bytes):
  compute_clover   links read once, 4 V 18 prec, plus A written, 72 V prec
  clover_invert    A read and A^-1 written, 2 x 72 V prec (the call also synchronises and copies two doubles back)
Flop model per site (an FMA counts 2):
  compute_clover   the reference's own counts: 6 planes x (12 SU(3) products x 198 + 54) (field_strength_tensor.cuh)
                   + 480 for the blocks (clover_compute.cuh)
  clover_invert    per 6x6 block in double: Cholesky 268 (incl. one sqrt, one division and one log per row), L^-1 310,
                   L^-dagger L^-1 448; two blocks per site

  python tools/bench_clover_build.py [--dim 32 32 32 32] [--reps 50] [--warmup 5]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

BUILD_FLOPS = 6 * (12 * 198 + 54) + 480
INVERT_FLOPS = 2 * (268 + 310 + 448)


def timed(fn, reps, warmup):
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
    return t0.elapsed_time(t1) * 1e3 / reps  # us per call


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dim", type=int, nargs=4, default=[32, 32, 32, 32])
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    import torch

    from quda_b200 import dslash as D
    from solver_bench import card
    assert torch.cuda.is_available(), "bench_clover_build.py measures on a CUDA device"
    X = a.dim
    V = X[0] * X[1] * X[2] * X[3]
    info = card()
    coeff = 0.12195 * 1.7
    for prec in (8, 4):
        dt = torch.float64 if prec == 8 else torch.float32
        # random links, unitarised: the construction does not care, but a positive-definite A keeps the Cholesky finite
        g = torch.linalg.qr(torch.randn((4, V, 3, 3), dtype=torch.complex128, device="cuda"))[0]
        gauge = torch.view_as_real(g).to(dt).contiguous()
        packed = torch.empty((V, 2, 36), dtype=dt, device="cuda")
        inv = torch.empty_like(packed)
        us = timed(lambda: D.compute_clover(packed, gauge, X, (0, 0, 0, 0), prec, coeff), a.reps, a.warmup)
        nbytes = (4 * 18 + 72) * V * prec
        print(json.dumps(dict(call="b200_compute_clover", dim=X, prec=prec, us_per_call=round(us, 2),
                              gbs=round(nbytes / us / 1e3, 1), gflops=round(BUILD_FLOPS * V / us / 1e3, 1),
                              bytes_model="4 V 18 prec + 72 V prec", flops_per_site=BUILD_FLOPS, card=info)))
        us = timed(lambda: D.clover_invert(inv, packed, X, prec), a.reps, a.warmup)
        nbytes = 2 * 72 * V * prec
        print(json.dumps(dict(call="b200_clover_invert_packed", dim=X, prec=prec, us_per_call=round(us, 2),
                              gbs=round(nbytes / us / 1e3, 1), gflops=round(INVERT_FLOPS * V / us / 1e3, 1),
                              bytes_model="2 x 72 V prec", flops_per_site=INVERT_FLOPS, card=info)))


if __name__ == "__main__":
    main()
