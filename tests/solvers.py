"""Shared harness of the single-GPU solver tests (CG, BiCGStab, multi-shift CG): the operators of a seeded Problem, the
invertQuda-style solve through prepare / reconstruct, and the host-side fp64 residuals from the oracle that every solution
is checked against."""
import contextlib
import ctypes as C

import numpy as np

import oracle
from common import CudaMem, Problem
from quda_b200 import dirac as DR
from quda_b200 import dslash as D
from quda_b200 import lib as L

KAPPA = 0.12195
MU = 0.1
X8 = (8, 8, 8, 8)
OFFSETS = [0.0, 1e-3, 1e-2, 0.1, 1.0, 10.0]  # multi-shift CG's shifts sigma_j

CASES = [
    ("wilsonpc", dict(), DR.MATPC_EVEN_EVEN),
    ("wilsonpc", dict(), DR.MATPC_ODD_ODD_ASYMMETRIC),
    ("cloverpc", dict(clover=True, compressed=True, dynamic=True), DR.MATPC_EVEN_EVEN),
    ("cloverpc", dict(clover=True, compressed=False, dynamic=False), DR.MATPC_EVEN_EVEN),
    ("cloverpc", dict(clover=True, compressed=False, dynamic=False), DR.MATPC_ODD_ODD_ASYMMETRIC),
    ("cloverpc", dict(clover=True, compressed=True, dynamic=True), DR.MATPC_EVEN_EVEN_ASYMMETRIC),
    ("twistedmasspc", dict(), DR.MATPC_EVEN_EVEN),
    ("twistedmasspc", dict(), DR.MATPC_ODD_ODD_ASYMMETRIC),
]
CASE_IDS = [f"{k}-{'dyn' if p.get('dynamic') else ('static' if p else 'plain')}-matpc{m}" for k, p, m in CASES]

# one rank: the global sum is the local one
_IDENTITY_ALLREDUCE = L.ALLREDUCE_FN(lambda data, n, user: None)


def operators(P, kind, matpc=DR.MATPC_EVEN_EVEN, kappa=KAPPA, mixed=False, stream=None, comm=None):
    """(precise, sloppy): the operator on P's fields and, if mixed, the same operator in single precision (recon 12,
    compressed dynamic clover) on a Problem of the same seeds, else None.  comm maps precision to a comm block."""
    kw = dict(clover=P.A, clover_inv=P.Ainv) if "clover" in kind else {}
    if kind.startswith("twistedmass"):
        kw["mu"] = MU
    precise = DR.Dirac(kind, P.U, kappa, matpc_type=matpc, stream=stream, comm=comm[8] if comm else None, **kw)
    if not mixed:
        return precise, None
    Ps = Problem(P.X, 4, 12, CudaMem, clover=P.clover is not None, compressed=True, dynamic=True)
    kws = dict(clover=Ps.A, clover_inv=Ps.Ainv) if "clover" in kind else {}
    if kind.startswith("twistedmass"):
        kws["mu"] = MU
    sloppy = DR.Dirac(kind, Ps.U, kappa, matpc_type=matpc, stream=stream, comm=comm[4] if comm else None, **kws)
    sloppy._keep = Ps
    return precise, sloppy


def full_residual(P, kind, x, b, kappa=KAPPA):
    """|M x - b| / |b| with the oracle's unpreconditioned operator, in float64"""
    x = x.astype(np.float64)
    if "clover" in kind:
        Mx = oracle.clover_mat(P.gauge, P.clover, x, P.X, kappa, 0)
    elif kind.startswith("twistedmass"):
        Mx = oracle.tm_mat(P.gauge, x, P.X, kappa, MU, 0)
    else:
        Mx = oracle.wil_mat(P.gauge, x, P.X, kappa, 0)
    return float(np.linalg.norm(Mx.astype(np.float64).ravel() - b.astype(np.float64).ravel()) / np.linalg.norm(b.ravel()))


def shift_residual(P, kind, matpc, x, b, sigma, kappa=KAPPA):
    """|(M^dag M + sigma) x - b| / |b| on the host in fp64 (the preconditioned operator for the *pc types, the full one
    otherwise)"""
    x = x.astype(np.float64)
    if kind == "wilsonpc":
        m = lambda v, d: oracle.wil_matpc(P.gauge, v, P.X, kappa, matpc, d)  # noqa: E731
    elif kind == "cloverpc":
        m = lambda v, d: oracle.clover_matpc(P.gauge, P.clover, P.clover_inv, v, P.X, kappa, matpc, d)  # noqa: E731
    elif kind == "twistedmasspc":
        m = lambda v, d: oracle.tm_matpc(P.gauge, v, P.X, kappa, MU, matpc, d)  # noqa: E731
    elif kind == "wilson":
        m = lambda v, d: oracle.wil_mat(P.gauge, v, P.X, kappa, d)  # noqa: E731
    else:
        m = lambda v, d: oracle.clover_mat(P.gauge, P.clover, v, P.X, kappa, d)  # noqa: E731
    r = m(m(x, 0), 1) + sigma * x - b.astype(np.float64)
    return float(np.linalg.norm(r.ravel()) / np.linalg.norm(b.ravel()))


def solve_prepared(precise, sloppy, solver, xdev, bdev, maxiter):
    """prepare -> CG on M_pc^dag M_pc (source M_pc^dag src) or BiCGStab on M_pc -> reconstruct, to 1e-10; xdev and bdev
    hold both parities.  Returns the solver result."""
    src_p, sol_p = precise.prepare(xdev, bdev)
    pb = xdev.parity_bytes
    src = D.ColorSpinorField(xdev.buf[src_p * pb:(src_p + 1) * pb], xdev.X, xdev.prec)
    sol = D.ColorSpinorField(xdev.buf[sol_p * pb:(sol_p + 1) * pb], xdev.X, xdev.prec)
    rhs = D.ColorSpinorField(CudaMem.empty(pb), xdev.X, xdev.prec)
    if solver == "cg":
        precise.Mdag(rhs, src)  # normal equations: M^dag M sol = M^dag src
    else:
        rhs.buf.copy_(src.buf)  # the source lives in x's other-parity half, which reconstruct overwrites
    sol.buf.zero_()
    invert = DR.invert_cg if solver == "cg" else DR.invert_bicgstab
    res = invert(precise, sloppy, sol, rhs, tol=1e-10, maxiter=maxiter)
    precise.reconstruct(xdev, bdev)
    return res


def solve(P, kind, solver, matpc=DR.MATPC_EVEN_EVEN, mixed=False, kappa=KAPPA, stream=None, comm=None):
    """M x = b from the seed-77 source: through prepare / reconstruct for the *pc types, BiCGStab on the full field
    otherwise.  Returns (solver result, host-verified full-system residual, solution, source)."""
    precise, sloppy = operators(P, kind, matpc, kappa, mixed, stream, comm)
    b = P.spinor(seed=77, nparity=2)
    bdev, xdev = P.to_dev(b, 2), P.empty(2)
    if kind.endswith("pc"):
        res = solve_prepared(precise, sloppy, solver, xdev, bdev, maxiter=2000)
    else:
        assert solver == "bicgstab", solver
        res = DR.invert_bicgstab(precise, sloppy, xdev, bdev, tol=1e-10, maxiter=2000)
    x = P.to_host(xdev)
    return res, full_residual(P, kind, x, b, kappa), x, b


def solve_multishift(P, kind, offsets, matpc=DR.MATPC_EVEN_EVEN, mixed=False, kappa=KAPPA, tol_offset=None, stream=None,
                     comm=None, b=None, xs=None, ops=None):
    """multi-shift solve to 1e-10 from b (default: the seed-77 source); returns (result, [x_j on the host], b on the host)"""
    precise, sloppy = ops or operators(P, kind, matpc, kappa, mixed, stream, comm)
    npar = 1 if kind.endswith("pc") else 2
    if b is None:
        b = P.spinor(seed=77, nparity=npar)
    bdev = P.to_dev(b, npar)
    if xs is None:
        xs = [P.empty(npar) for _ in offsets]
    res = DR.invert_multishift_cg(precise, sloppy, xs, bdev, offsets, tol=1e-10, tol_offset=tol_offset, maxiter=2000)
    return res, [P.to_host(x) for x in xs], b


def check_shifts(P, kind, matpc, res, xs, b, offsets, tols, kappa=KAPPA, bound=1e-8):
    for j, (sigma, x) in enumerate(zip(offsets, xs)):
        assert np.isfinite(x).all(), j
        rr = shift_residual(P, kind, matpc, x, b, sigma, kappa)
        assert rr < bound, (j, sigma, rr)
        assert res.true_res_offset[j] <= tols[j], (j, res.true_res_offset[j], tols[j])
        assert np.isfinite(res.iter_res_offset[j]), j
        assert 0 <= res.iter_offset[j] <= res.iter, (j, res.iter_offset[j], res.iter)


def self_exchanges(X):
    """one GPU that is its own neighbour in every dimension: {prec: HaloExchange} and {prec: comm block} for the fp64
    and fp32 operators"""
    from quda_b200 import comm
    grid = comm.ProcessGrid((1, 1, 1, 1), 0)
    exs = {p: comm.HaloExchange(grid, X, p, mode="self") for p in (8, 4)}
    return exs, {p: e.comm_struct() for p, e in exs.items()}


def set_host_allreduce(css, on):
    """With no mailbox ranks and an identity callback set, every global sum of the solve goes through the host."""
    for cs in css.values():
        assert cs.n_ranks == 0  # no mailboxes: with a callback set, every sum goes through it
        cs.allreduce_sum = C.cast(_IDENTITY_ALLREDUCE, C.c_void_p) if on else None


@contextlib.contextmanager
def busy_default_stream():
    """Yields a fresh side stream (cudaStreamNonBlocking: it does NOT synchronise with the legacy default stream) made
    current while the default stream is kept busy with unrelated work; synchronises it on the way out."""
    import torch
    side = torch.cuda.Stream()
    junk = torch.empty(64 << 20, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    for _ in range(20):
        junk.add_(1.0)
    with torch.cuda.stream(side):
        yield side
        side.synchronize()
