"""GPU tier: multi-shift CG (b200_invert_multishift_cg, lib/inv_multi_cg_quda.cpp) on (MdagM + sigma_j) x_j = b for the Wilson,
clover and twisted-mass operators.  Every shifted solution is checked on the host in fp64 with the oracle's operator
(M_pc^dag M_pc from *_matpc with dagger 0 then 1, or the full M^dag M), so a wrong zeta / alpha / beta recursion, a shift
update that pairs the wrong fields, or a shift that retires too early shows up as a residual, not just as an iteration
count."""
import ctypes as C

import numpy as np
import pytest

from common import CudaMem, Problem
from quda_b200 import dirac as DR
from quda_b200 import lib as L
from solvers import (CASE_IDS, CASES, KAPPA, OFFSETS, X8, busy_default_stream, check_shifts, operators, self_exchanges,
                     set_host_allreduce, shift_residual, solve_multishift)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("mixed", [False, True], ids=["fp64", "fp64-fp32"])
@pytest.mark.parametrize("kind,pkw,matpc", CASES, ids=CASE_IDS)
def test_multishift_preconditioned_system(kind, pkw, matpc, mixed):
    P = Problem(X8, 8, 18, CudaMem, **pkw)
    res, xs, b = solve_multishift(P, kind, OFFSETS, matpc, mixed)
    assert 0 < res.iter < 2000, res.iter
    check_shifts(P, kind, matpc, res, xs, b, OFFSETS, [1e-10] * len(OFFSETS))
    if mixed:
        assert res.reliable_updates >= 1, res.reliable_updates
    else:
        assert res.reliable_updates == 0
        assert list(res.refine_iter[:len(OFFSETS)]) == [0] * len(OFFSETS)  # fp64 alone needs no refinement


@pytest.mark.parametrize("kind", ["wilson", "clover"])
def test_multishift_full_system(kind):
    P = Problem(X8, 8, 18, CudaMem, clover=kind == "clover", compressed=True, dynamic=True)
    res, xs, b = solve_multishift(P, kind, OFFSETS)
    check_shifts(P, kind, None, res, xs, b, OFFSETS, [1e-10] * len(OFFSETS))


@pytest.mark.parametrize("mixed", [False, True], ids=["fp64", "fp64-fp32"])
def test_multishift_is_cheaper_than_sequential_solves(mixed):
    """one recursion for all shifts (plus its refinements) against one single-shift solve per shift"""
    P = Problem(X8, 8, 18, CudaMem, clover=True, compressed=True, dynamic=True)
    ops = operators(P, "cloverpc", DR.MATPC_EVEN_EVEN, mixed=mixed)
    ms, xs, b = solve_multishift(P, "cloverpc", OFFSETS, ops=ops)
    seq = 0
    for j, sigma in enumerate(OFFSETS):
        one, (x1,), _ = solve_multishift(P, "cloverpc", [sigma], b=b, ops=ops)
        assert shift_residual(P, "cloverpc", DR.MATPC_EVEN_EVEN, x1, b, sigma) < 1e-8
        seq += one.iter + one.refine_iter[0]
    total = ms.iter + sum(ms.refine_iter[:len(OFFSETS)])
    print(f"multi-shift {ms.iter} + refinement {list(ms.refine_iter[:len(OFFSETS)])} vs sequential {seq}")
    # with a single-precision sloppy operator the shifted solutions drift from their recursions and need refinement
    assert total < (0.75 if mixed else 0.5) * seq, (ms.iter, list(ms.refine_iter[:len(OFFSETS)]), seq)


def test_shift_zero_agrees_with_cg():
    P = Problem(X8, 8, 18, CudaMem, clover=True, compressed=True, dynamic=True)
    precise, _ = operators(P, "cloverpc", DR.MATPC_EVEN_EVEN)
    ms, xs, b = solve_multishift(P, "cloverpc", [0.0, 0.01, 0.1], ops=(precise, None))
    x = P.empty()
    cg = DR.invert_cg(precise, None, x, P.to_dev(b), tol=1e-10, maxiter=2000)
    x_cg = P.to_host(x)
    assert abs(ms.iter - cg.iter) <= 1, (ms.iter, cg.iter)
    assert ms.iter_offset[0] == ms.iter
    assert np.linalg.norm(xs[0] - x_cg) / np.linalg.norm(x_cg) < 1e-7
    assert shift_residual(P, "cloverpc", DR.MATPC_EVEN_EVEN, xs[0], b, 0.0) < 1e-8


def test_per_shift_tolerances_retire_shifts_early():
    P = Problem(X8, 8, 18, CudaMem, clover=True, compressed=True, dynamic=True)
    offsets = [0.0, 0.01, 0.1, 1.0]
    tight, _, _ = solve_multishift(P, "cloverpc", offsets)
    loose_tols = [1e-10, 1e-10, 1e-4, 1e-4]
    loose, xs, b = solve_multishift(P, "cloverpc", offsets, tol_offset=loose_tols)
    check_shifts(P, "cloverpc", DR.MATPC_EVEN_EVEN, loose, xs, b, offsets, loose_tols, bound=1.0)
    for j in (0, 1):
        assert shift_residual(P, "cloverpc", DR.MATPC_EVEN_EVEN, xs[j], b, offsets[j]) < 1e-8
    for j in (2, 3):
        assert loose.iter_offset[j] < tight.iter_offset[j], (j, list(loose.iter_offset[:4]), list(tight.iter_offset[:4]))
        assert loose.iter_offset[j] < loose.iter_offset[0]
        assert shift_residual(P, "cloverpc", DR.MATPC_EVEN_EVEN, xs[j], b, offsets[j]) < 2e-4
    assert loose.iter_offset[3] <= loose.iter_offset[2] <= loose.iter_offset[1] <= loose.iter_offset[0] == loose.iter


def test_zero_source_gives_zero_solutions():
    P = Problem(X8, 8, 18, CudaMem)
    xs = [P.to_dev(P.spinor(seed=5 + j)) for j in range(3)]  # non-zero on entry
    res, out, _ = solve_multishift(P, "wilsonpc", [0.0, 0.1, 1.0], b=np.zeros_like(P.spinor()), xs=xs)
    assert res.iter == 0
    for x in out:
        assert not x.any()


def test_kappa_zero_one_iteration():
    """kappa = 0: M_pc = 1, so (1 + sigma_j) x_j = b is solved by the first iteration: x_j = alpha_j b with
    alpha_j = 1 / (1 + sigma_j) from the zeta recursion"""
    P = Problem(X8, 8, 18, CudaMem)
    offsets = [0.0, 1e-3, 0.1, 1.0, 10.0]
    res, xs, b = solve_multishift(P, "wilsonpc", offsets, kappa=0.0)
    assert res.iter == 1, res.iter
    b_dev = P.to_host(P.to_dev(b))  # the native order is a rotated gamma basis: compare with b as the device holds it
    for j, sigma in enumerate(offsets):
        assert np.isfinite(xs[j]).all() and np.isfinite(res.iter_res_offset[j]), j
        want = b_dev / (1.0 + sigma)
        assert np.linalg.norm(xs[j] - want) / np.linalg.norm(want) < 1e-14, j
        assert res.iter_offset[j] == 1 and res.refine_iter[j] == 0


@pytest.mark.parametrize("n", [1, 32])
def test_one_and_thirty_two_shifts(n):
    P = Problem(X8, 8, 18, CudaMem, clover=True, compressed=True, dynamic=True)
    offsets = [0.05] if n == 1 else [0.0] + list(np.geomspace(1e-4, 10.0, n - 1))
    res, xs, b = solve_multishift(P, "cloverpc", offsets, mixed=True)
    check_shifts(P, "cloverpc", DR.MATPC_EVEN_EVEN, res, xs, b, offsets, [1e-10] * n)


def test_duplicate_offsets():
    P = Problem(X8, 8, 18, CudaMem, clover=True, compressed=True, dynamic=True)
    offsets = [0.0, 0.1, 0.1, 1.0, 1.0]
    res, xs, b = solve_multishift(P, "cloverpc", offsets)
    check_shifts(P, "cloverpc", DR.MATPC_EVEN_EVEN, res, xs, b, offsets, [1e-10] * len(offsets))
    assert np.array_equal(xs[1], xs[2]) and np.array_equal(xs[3], xs[4])


def test_initial_guess_is_ignored():
    P = Problem(X8, 8, 18, CudaMem, clover=True, compressed=True, dynamic=True)
    ops = operators(P, "cloverpc", DR.MATPC_EVEN_EVEN, mixed=True)
    ref, x_ref, b = solve_multishift(P, "cloverpc", OFFSETS, ops=ops)
    dirty = [P.to_dev(P.spinor(seed=100 + j)) for j in range(len(OFFSETS))]
    res, xs, _ = solve_multishift(P, "cloverpc", OFFSETS, ops=ops, b=b, xs=dirty)
    assert res.iter == ref.iter
    for a, c in zip(xs, x_ref):
        assert np.array_equal(a, c)


def test_multishift_is_bit_reproducible():
    P = Problem(X8, 8, 18, CudaMem, clover=True, compressed=True, dynamic=True)
    a = solve_multishift(P, "cloverpc", OFFSETS, mixed=True)
    c = solve_multishift(P, "cloverpc", OFFSETS, mixed=True)
    assert a[0].iter == c[0].iter and list(a[0].true_res_offset) == list(c[0].true_res_offset)
    for x, y in zip(a[1], c[1]):
        assert np.array_equal(x, y)


def _sync_bound(res, n, host_waits=1):
    return host_waits * (res.iter + sum(res.refine_iter[:n])) + 4 * (res.reliable_updates + n + 2)


@pytest.mark.parametrize("mixed", [False, True], ids=["fp64", "fp64-fp32"])
def test_host_allreduce_matches_the_device_path(mixed):
    """a self-partitioned exchange with an identity callback and no mailbox ranks sends every global sum through the host;
    the host derives the scalars with the same function the finalisers run"""
    P = Problem(X8, 8, 12, CudaMem, clover=True, compressed=True, dynamic=True)
    exs, css = self_exchanges(P.X)
    n = len(OFFSETS)
    out = {}
    for callback in (False, True):
        set_host_allreduce(css, callback)
        res, xs, b = solve_multishift(P, "cloverpc", OFFSETS, mixed=mixed, comm=css)
        check_shifts(P, "cloverpc", DR.MATPC_EVEN_EVEN, res, xs, b, OFFSETS, [1e-10] * n)
        assert res.host_syncs <= _sync_bound(res, n, 2 if callback else 1), (callback, res.host_syncs, res.iter)
        assert not any(e.timed_out() for e in exs.values())
        out[callback] = (res, xs)
    if mixed:
        return
    (dev, x_dev), (host, x_host) = out[False], out[True]
    assert dev.iter == host.iter, (dev.iter, host.iter)
    assert list(dev.iter_offset[:n]) == list(host.iter_offset[:n])
    for a, c in zip(x_dev, x_host):
        assert np.array_equal(a, c)


@pytest.mark.parametrize("mixed", [False, True], ids=["fp64", "fp64-fp32"])
def test_multishift_on_a_non_blocking_stream(mixed):
    """every kernel on the operator's stream while the default stream is kept busy; the host follows one iteration behind"""
    P = Problem(X8, 8, 18, CudaMem, clover=True, compressed=True, dynamic=True)
    with busy_default_stream() as side:
        res, xs, b = solve_multishift(P, "cloverpc", OFFSETS, mixed=mixed, stream=side.cuda_stream)
    check_shifts(P, "cloverpc", DR.MATPC_EVEN_EVEN, res, xs, b, OFFSETS, [1e-10] * len(OFFSETS))
    assert res.host_syncs <= _sync_bound(res, len(OFFSETS)), (res.host_syncs, res.iter, res.reliable_updates)


def test_multishift_self_partitioned():
    """one GPU that is its own neighbour in every dimension: every Dslash goes through pack + ghost, one exchange per
    precision"""
    P = Problem(X8, 8, 12, CudaMem, clover=True, compressed=True, dynamic=True)
    exs, css = self_exchanges(P.X)
    res, xs, b = solve_multishift(P, "cloverpc", OFFSETS, mixed=True, comm=css)
    check_shifts(P, "cloverpc", DR.MATPC_EVEN_EVEN, res, xs, b, OFFSETS, [1e-10] * len(OFFSETS))
    assert res.reliable_updates >= 1
    assert not any(e.timed_out() for e in exs.values())


def test_multishift_argument_checks():
    import torch
    lib = L.load()
    P = Problem((4, 4, 4, 4), 8, 18, CudaMem)
    op = DR.Dirac("wilsonpc", P.U, KAPPA)
    b = P.to_dev(P.spinor(seed=3))
    xs = [P.empty() for _ in range(3)]

    def refused(sloppy, match, precise=op, x=xs, bf=b, offsets=(0.0, 0.1, 1.0)):
        with pytest.raises(L.B200Error, match=match):
            DR.invert_multishift_cg(precise, sloppy, x, bf, list(offsets), maxiter=10)

    Ph = Problem((4, 4, 4, 4), 2, 12, CudaMem)
    refused(DR.Dirac("wilsonpc", Ph.U, KAPPA), "double or single")
    Ps = Problem((4, 4, 4, 4), 4, 12, CudaMem)
    side = torch.cuda.Stream()
    refused(DR.Dirac("wilsonpc", Ps.U, KAPPA, stream=side.cuda_stream), "share a stream")
    refused(None, "precision", x=[xs[0], Ps.empty(), xs[2]])
    refused(None, "precision", bf=Ps.to_dev(Ps.spinor(seed=3)))
    refused(None, "non-decreasing", offsets=(0.0, 1.0, 0.1))

    # the same refusals from the library itself, past the wrapper
    def lib_refuses(match, n=3, offsets=(0.0, 0.1, 1.0), x=xs, bf=b):
        p = L.MultiShiftParam()
        p.n_shift, p.maxiter = n, 10
        for j, o in enumerate(offsets):
            p.offset[j], p.tol_offset[j] = o, 1e-10
        xd = (L.Spinor * L.MAX_SHIFTS)(*[f.desc() for f in (list(x) * L.MAX_SHIFTS)[:L.MAX_SHIFTS]])
        bd = bf.desc()
        assert lib.b200_invert_multishift_cg(op.h, None, xd, C.byref(bd), C.byref(p)) == -1
        assert match in lib.b200_last_error()

    lib_refuses(b"n_shift 0", n=0)
    lib_refuses(b"n_shift 33", n=33)
    lib_refuses(b"non-decreasing", offsets=(0.0, 1.0, 0.1))
    lib_refuses(b"distinct", x=[xs[0], xs[0], xs[2]])
