"""GPU tier: b200_compute_clover / b200_clover_invert_packed against the numpy restatement (tests/clover_build_ref.py) and,
in fp64, bit for bit against the host twin of the same site code; dslash.compute_clover_field end to end through mixed
double/single clover-PC solves checked on the host with the oracle's full operator; the free field; two GPUs through
comm.extend_gauge."""
import numpy as np
import pytest
import torch

import clover_build_ref as R
import oracle
from clover_twin import clover_twin
from common import CudaMem, Problem, assert_close
from quda_b200 import dirac as DR
from quda_b200 import dslash as D
from quda_b200 import fields as F
from solvers import KAPPA, full_residual, solve_prepared

pytestmark = pytest.mark.gpu

CSW = 1.7
TOL = {8: 1e-13, 4: 1e-5}


def gpu_clover(gauge, X, coeff, prec):
    g = torch.from_numpy(gauge).cuda()
    packed = torch.empty((int(np.prod(X)), 2, 36), dtype=g.dtype, device="cuda")
    D.compute_clover(packed, g, X, (0, 0, 0, 0), prec, coeff)
    inv = torch.empty_like(packed)
    tl = D.clover_invert(inv, packed, X, prec)
    return packed.cpu().numpy(), inv.cpu().numpy(), tl


@pytest.mark.parametrize("X", [(8, 8, 8, 8), (16, 16, 16, 16)])
@pytest.mark.parametrize("prec", [8, 4])
def test_library_matches_reference_and_twin(X, prec):
    coeff = KAPPA * CSW
    gauge = oracle.random_gauge(X, prec, seed=31)
    A, inv, tl = gpu_clover(gauge, X, coeff, prec)
    A64 = A.astype(np.float64)
    assert np.abs(A - R.compute_clover(gauge.astype(np.float64), X, coeff)).max() <= TOL[prec]
    want_inv, _ = R.invert(A64)
    assert np.abs(inv - want_inv).max() <= TOL[prec]
    assert np.allclose(tl, R.trlog(A64), rtol=1e-12, atol=1e-9)
    assert gpu_clover(gauge, X, coeff, prec)[2] == tl  # fixed-order reduction: bit-identical sums
    if prec == 8:  # the site code rounds identically on the device and in the host twin
        tA = np.zeros_like(A)
        D.compute_clover(tA, gauge, X, (0, 0, 0, 0), 8, coeff, backend=clover_twin())
        assert np.array_equal(A, tA)
        tinv = np.zeros_like(A)
        D.clover_invert(tinv, tA, X, 8, backend=clover_twin())
        assert np.array_equal(inv, tinv)


@pytest.mark.parametrize("compressed,dynamic", [(True, True), (False, False)], ids=["compressed-dynamic", "static-inverse"])
@pytest.mark.parametrize("solver", ["cg", "bicgstab"])
def test_compute_clover_field_solves(compressed, dynamic, solver):
    """even-even clover-PC, mixed double / single, to 1e-10 with the computed clover term; the full-system residual uses the
    oracle's operator on the reference clover term"""
    X = (8, 8, 8, 8)
    P = Problem(X, 8, 18, CudaMem)
    A8, Ai8, _ = D.compute_clover_field(P.gauge, X, 8, KAPPA, CSW, compressed=compressed, dynamic=dynamic)
    Ps = Problem(X, 4, 12, CudaMem)
    A4, Ai4, _ = D.compute_clover_field(Ps.gauge, X, 4, KAPPA, CSW, compressed=True, dynamic=True)
    precise = DR.Dirac("cloverpc", P.U, KAPPA, clover=A8, clover_inv=Ai8)
    sloppy = DR.Dirac("cloverpc", Ps.U, KAPPA, clover=A4, clover_inv=Ai4)
    P.clover = R.compute_clover(P.gauge, X, KAPPA * CSW)  # what full_residual's oracle operator uses
    b = P.spinor(seed=77, nparity=2)
    bdev, xdev = P.to_dev(b, 2), P.empty(2)
    res = solve_prepared(precise, sloppy, solver, xdev, bdev, maxiter=2000)
    assert res.iter < 2000 and res.true_res < 5e-10, (res.iter, res.true_res)
    assert full_residual(P, "cloverpc", P.to_host(xdev), b) < 1e-8


@pytest.mark.parametrize("prec", [8, 4, 2])
def test_compute_clover_field_applies_as_reference(prec):
    """compressed A at every precision, half included: ApplyClover with the computed field == oracle.apply_clover with the
    reference clover term"""
    X = (8, 8, 8, 8)
    P = Problem(X, prec, 18, CudaMem)
    A, _, tl = D.compute_clover_field(P.gauge, X, prec, KAPPA, CSW, compressed=True, dynamic=True)
    ref = R.compute_clover(P.gauge.astype(np.float64), X, KAPPA * CSW)
    assert np.allclose(tl, R.trlog(ref), rtol=1e-5)
    for parity in range(2):
        s = P.spinor(seed=9 + parity)
        out = P.empty()
        D.ApplyClover(out, P.to_dev(s), A, False, parity)
        assert_close(oracle.apply_clover(ref.astype(P.gauge.dtype), s, X, parity), P.to_host(out), prec, 18, "computed clover")


@pytest.mark.parametrize("free", ["csw0", "unit-links"])
def test_free_field_is_wilson(free):
    """csw = 0, or unit links (F = 0): A = 1 and the clover operator is the Wilson operator"""
    X = (8, 8, 8, 8)
    P = Problem(X, 8, 18, CudaMem)
    if free == "unit-links":
        P.gauge = np.zeros_like(P.gauge)
        for c in range(3):
            P.gauge[:, :, c, c, 0] = 1.0
        gbuf, gmeta = F.gauge_to_native(P.gauge, X, 8, 18)
        P.U = D.GaugeField(CudaMem.put(gbuf), X, 8, 18, gmeta, t_boundary=-1)
    A, _, tl = D.compute_clover_field(P.gauge, X, 8, KAPPA, 0.0 if free == "csw0" else CSW)
    assert tl == [0.0, 0.0]
    s = P.spinor(seed=4, nparity=2)
    out_c, out_w = P.empty(2), P.empty(2)
    DR.Dirac("clover", P.U, KAPPA, clover=A).M(out_c, P.to_dev(s, 2))
    DR.Dirac("wilson", P.U, KAPPA).M(out_w, P.to_dev(s, 2))
    assert_close(P.to_host(out_w), P.to_host(out_c), 8, 18, "free clover vs Wilson")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_two_gpus_extend_gauge():
    from clover_build_worker import worker
    from dist_worker import run_ranks
    for r in run_ranks(worker, 2, ((1, 1, 1, 2), (8, 8, 8, 8), "gpu"), timeout=600):
        assert r["dev"] <= 1e-13, (r["rank"], r["dev"])
        assert np.allclose(r["trlog"], r["trlog_ref"], rtol=0, atol=1e-9), r
