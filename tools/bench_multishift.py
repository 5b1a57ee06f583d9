#!/usr/bin/env python
"""Time multi-shift CG against one single-shift solve per shift on an RHMC-like pole set: Wilson-clover, symmetric even-even
preconditioning, double precision with a single-precision sloppy operator and reliable updates (--sloppy double: double
throughout), global lattice --global-dim (default 32^3 x 64) split over the ranks.  The system is
(M_pc^dag M_pc + sigma_j) x_j = b.

  python tools/bench_multishift.py [--global-dim X Y Z T] [--tol 1e-10] [--reps 1] [--sloppy single|double] [--no-xp]
  torchrun --nproc-per-node N tools/bench_multishift.py ...

Each mode gets one warm-up, then the two are timed alternately with CUDA events:
  multishift   one invert_multishift_cg over all offsets (with its refinement)
  sequential   one single-shift invert_multishift_cg per offset, i.e. CG on M_pc^dag M_pc + sigma_j
One JSON line per mode: iterations, M_pc^dag M_pc applications (counted from the solver's statistics), refinement
iterations, time to solution, the per-shift true residual, and the card and its power limit.

Then one line for the shift update kernel ms_update_xp (fp32, the sloppy precision) at n_active = 1, 4, 12, 32: a solve with
n equal offsets keeps all n shifts active, its kernel durations come from torch.profiler's CUDA kernel records, and the
achieved bandwidth uses the (1 + 4 n) S byte model (S = one single-parity fp32 spinor field) against the H100 SXM data
sheet's 3.35 TB/s."""
import argparse
import json
import statistics

from solver_bench import card, max_over_ranks, setup, timed_runs

# 12 poles over 1e-4 .. 10, as a rational approximation for RHMC has them
OFFSETS = [1e-4 * (1e5 ** (j / 11)) for j in range(12)]
HBM_GBS = 3350.0


def mdagm_applications(res, n):
    """M_pc^dag M_pc applications of one invert_multishift_cg call: one per iteration, one for the iteration queued behind
    the converged one, the initial residual, one per reliable update and one true residual per shift; each refinement adds
    its iterations and the same three fixed ones"""
    refined = sum(1 for j in range(n) if res.refine_iter[j] > 0)
    return res.iter + sum(res.refine_iter[:n]) + res.reliable_updates + 2 + n + 3 * refined


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--global-dim", type=int, nargs=4, default=[32, 32, 32, 64])
    ap.add_argument("--tol", type=float, default=1e-10)
    ap.add_argument("--kappa", type=float, default=0.12195)
    ap.add_argument("--reps", type=int, default=1, help="timed solves per mode (alternating)")
    ap.add_argument("--sloppy", choices=["single", "double"], default="single")
    ap.add_argument("--xp-iters", type=int, default=20, help="multi-shift iterations per shift-update measurement")
    ap.add_argument("--no-xp", action="store_true", help="skip the shift-update kernel measurement")
    a = ap.parse_args()

    import torch
    from quda_b200 import dirac as DR, dslash as D, fields as F
    rank, world, dist, dims, X, ops = setup(a.global_dim, a.kappa)
    Xg = a.global_dim
    pc = ops[8]
    sloppy = ops[4] if a.sloppy == "single" else None
    pb = F.spinor_bytes(X, 8)
    g = torch.Generator(device="cuda").manual_seed(99 + rank)
    b = D.ColorSpinorField(torch.rand(pb // 8, dtype=torch.float64, device="cuda", generator=g).view(torch.uint8), X, 8)

    def fields(n):
        return [D.ColorSpinorField(torch.zeros(pb, dtype=torch.uint8, device="cuda"), X, 8) for _ in range(n)]

    xs = fields(len(OFFSETS))

    def solve(mode):
        if mode == "multishift":
            return [DR.invert_multishift_cg(pc, sloppy, xs, b, OFFSETS, tol=a.tol, maxiter=20000)]
        return [DR.invert_multishift_cg(pc, sloppy, [x], b, [s], tol=a.tol, maxiter=20000) for s, x in zip(OFFSETS, xs)]

    modes = ("multishift", "sequential")
    runs = {m: [] for m in modes}
    for m, secs, res in timed_runs(modes, solve, a.reps, dist):
        runs[m].append((secs, res))
    info = card()
    for m in modes:
        secs, res = min(runs[m], key=lambda r: r[0])
        secs, = max_over_ranks(dist, secs)
        if m == "multishift":
            r, n = res[0], len(OFFSETS)
            iters, refine = r.iter, list(r.refine_iter[:n])
            true_res, rel = list(r.true_res_offset[:n]), r.reliable_updates
            mdagm = mdagm_applications(r, n)
        else:
            iters, refine = sum(r.iter for r in res), [r.refine_iter[0] for r in res]
            true_res, rel = [r.true_res_offset[0] for r in res], sum(r.reliable_updates for r in res)
            mdagm = sum(mdagm_applications(r, 1) for r in res)
        out = {"mode": m, "system": "(M_pc^dag M_pc + sigma_j) x_j = b", "offsets": OFFSETS, "iterations": iters,
               "refinement_iterations": refine, "mdagm_applications": mdagm, "reliable_updates": rel,
               "time_to_solution_s": secs, "true_res_offset": true_res, "timed_solves": len(runs[m]),
               "global_dim": Xg, "grid": dims, "n_gpus": world, "tol": a.tol, "kappa": a.kappa,
               "precision": "double recon-18 / " + ("single recon-12 sloppy" if sloppy else "no sloppy operator"), "card": info["name"],
               "power_limit_w": info["power_limit_w"]}
        if rank == 0:
            print(json.dumps(out), flush=True)
    del xs
    if not a.no_xp:
        # the shift update alone: n equal offsets keep all n shifts active for the whole solve
        S = F.spinor_bytes(X, 4)
        xp = []
        for n in (1, 4, 12, 32):
            xn = fields(n)
            DR.invert_multishift_cg(pc, ops[4], xn, b, [0.01] * n, tol=a.tol, maxiter=3)  # warm-up
            torch.cuda.synchronize()
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                res = DR.invert_multishift_cg(pc, ops[4], xn, b, [0.01] * n, tol=a.tol, maxiter=a.xp_iters)
                torch.cuda.synchronize()
            # the first `iter` updates belong to the multi-shift loop (any refinement solves come after it, with one shift)
            ev = sorted((e for e in prof.events() if "ms_update_xp_kernel" in e.name), key=lambda e: e.time_range.start)
            us = [e.time_range.elapsed_us() for e in ev[:res.iter]][2:]
            t = statistics.median(us) * 1e-6 if us else float("nan")
            nbytes = (1 + 4 * n) * S
            xp.append({"n_active": n, "calls": len(us), "median_us": t * 1e6, "bytes": nbytes, "gbs": nbytes / t * 1e-9,
                       "fraction_of_hbm": nbytes / t * 1e-9 / HBM_GBS})
            del xn
        if rank == 0:
            print(json.dumps({"kernel": "ms_update_xp", "precision": "single", "local_dim": X, "field_bytes": S, "runs": xp,
                              "hbm_gbs_reference": HBM_GBS, "card": info["name"], "power_limit_w": info["power_limit_w"]}),
                  flush=True)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
