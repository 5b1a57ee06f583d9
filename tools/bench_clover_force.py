#!/usr/bin/env python
"""Time the clover force on one GPU at 32^4 (--dim), fp64 and fp32, with n = 1 and 12 vectors.  One JSON line per kernel of
b200_clover_force_accumulate (microseconds from torch.profiler's CUDA activity over --reps calls after --warmup calls,
algorithmic bytes from the shapes below, GB/s and the fraction of 3.35 TB/s, the H100 SXM data-sheet HBM3 bandwidth), one
line for the whole call (CUDA events), and in fp64 one line with the end-to-end dirac.compute_clover_force next to one
12-pole multi-shift solve of the same system, for context.  The card's name and power limit are read in the same run.
The force is not a bandwidth-critical path: there is no speed target.

Byte model (prec = 8 or 4 bytes, V sites, n vectors):
  clover_hop_force_kernel   x and p read once, 2 n 24 V prec; links 4 18 V prec; mom read and written, 2 4 10 V prec
  clover_sigma_kernel       x and p read once, 2 n 24 V prec; A on the tr log parity, 72 V/2 prec; oprod written, 6 18 V prec
  clover_deriv_kernel       links 4 18 V prec; oprod read once, 6 18 V prec; mom read and written, 2 4 10 V prec

  python tools/bench_clover_force.py [--dim 32 32 32 32] [--reps 50] [--warmup 5]"""
import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

HBM = 3.35e12
KERNELS = {
    "clover_hop_force_kernel": lambda V, n, p: (2 * n * 24 + 4 * 18 + 2 * 4 * 10) * V * p,
    "clover_sigma_kernel": lambda V, n, p: (2 * n * 24 + 6 * 18) * V * p + 72 * V // 2 * p,
    "clover_deriv_kernel": lambda V, n, p: (4 * 18 + 6 * 18 + 2 * 4 * 10) * V * p,
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dim", type=int, nargs=4, default=[32, 32, 32, 32])
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    from quda_b200 import dirac as DR
    from quda_b200 import dslash as D
    from quda_b200 import fields as F
    from quda_b200 import lib as L
    from solver_bench import card
    assert torch.cuda.is_available(), "bench_clover_force.py measures on a CUDA device"
    X = a.dim
    V = X[0] * X[1] * X[2] * X[3]
    info = card()
    lib = L.load()
    kappa, csw = 0.12, 1.0
    g = torch.linalg.qr(torch.randn((4, V, 3, 3), dtype=torch.complex128, device="cuda"))[0]
    for prec in (8, 4):
        dt = torch.float64 if prec == 8 else torch.float32
        gauge = torch.view_as_real(g).to(dt).contiguous()
        packed = torch.empty((V, 2, 36), dtype=dt, device="cuda")
        D.compute_clover(packed, gauge, X, (0, 0, 0, 0), prec, kappa * csw)
        q = (C.c_void_p * 4)(*[gauge[mu].data_ptr() for mu in range(4)])
        for n in (1, 12):
            xs = [torch.randn(V * 24, dtype=dt, device="cuda") for _ in range(n)]
            ps = [torch.randn(V * 24, dtype=dt, device="cuda") for _ in range(n)]
            mom = torch.zeros((V, 4, 10), dtype=dt, device="cuda")
            xa = (C.c_void_p * n)(*[t.data_ptr() for t in xs])
            pa = (C.c_void_p * n)(*[t.data_ptr() for t in ps])
            fc = (C.c_double * n)(*([1e-3] * n))
            eps = (C.c_double * (2 * n))(*([1e-3] * (2 * n)))

            def call():
                L.check(lib.b200_clover_force_accumulate(mom.data_ptr(), q, packed.data_ptr(), (C.c_int * 4)(*X), prec, n, xa,
                                                         pa, fc, eps, 1e-3, 1, None))
            for _ in range(a.warmup):
                call()
            torch.cuda.synchronize()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(a.reps):
                call()
            t1.record()
            t1.synchronize()
            us_call = t0.elapsed_time(t1) * 1e3 / a.reps
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(a.reps):
                    call()
                torch.cuda.synchronize()
            for name, model in KERNELS.items():
                evs = [e for e in prof.events() if e.device_type.name == "CUDA" and name in e.name]
                us = sum(e.device_time for e in evs) / max(1, len(evs))
                nbytes = model(V, n, prec)
                print(json.dumps(dict(kernel=name, dim=X, prec=prec, n=n, launches=len(evs), us=round(us, 2),
                                      bytes=nbytes, gbs=round(nbytes / us / 1e3, 1), hbm_fraction=round(nbytes / us / 1e-6 / HBM, 3),
                                      card=info)))
            print(json.dumps(dict(call="b200_clover_force_accumulate", dim=X, prec=prec, n=n, us_per_call=round(us_call, 2),
                                  card=info)))
            del xs, ps
    # end to end in fp64, next to one 12-pole multi-shift solve of the same system
    from common import CudaMem  # noqa: E402  (tests/common.py: torch-backed device buffers)
    gauge = torch.view_as_real(g).contiguous()
    gbuf, gmeta = F.gauge_to_native(gauge.cpu().numpy(), X, 8, 18)
    U = D.GaugeField(CudaMem.put(gbuf), X, 8, 18, gmeta)
    A, Ainv, _ = D.compute_clover_field(gauge, X, 8, kappa, csw)
    op = DR.Dirac("cloverpc", U, kappa, clover=A, clover_inv=Ainv, matpc_type=DR.MATPC_EVEN_EVEN_ASYMMETRIC)
    nb = F.spinor_bytes(X, 8)
    b = D.ColorSpinorField(torch.randn(nb // 8, dtype=torch.float64, device="cuda"), X, 8)
    xs = [D.ColorSpinorField(torch.zeros(nb // 8, dtype=torch.float64, device="cuda"), X, 8) for _ in range(12)]
    offsets = [1e-4 * 3 ** j for j in range(12)]
    torch.cuda.synchronize()
    t = time.perf_counter()
    p = DR.invert_multishift_cg(op, None, xs, b, offsets, tol=1e-10)
    torch.cuda.synchronize()
    solve_ms = (time.perf_counter() - t) * 1e3
    mom = torch.zeros((V, 4, 10), dtype=torch.float64, device="cuda")
    DR.compute_clover_force(mom, 0.1, xs, [1.0] * 12, kappa, csw, 1, gauge, op)  # warm-up
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(3):
        DR.compute_clover_force(mom, 0.1, xs, [1.0] * 12, kappa, csw, 1, gauge, op)
    torch.cuda.synchronize()
    force_ms = (time.perf_counter() - t) * 1e3 / 3
    print(json.dumps(dict(call="compute_clover_force", dim=X, prec=8, n=12, ms=round(force_ms, 2),
                          multishift_12_ms=round(solve_ms, 1), multishift_iter=p.iter, card=info)))


if __name__ == "__main__":
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    main()
