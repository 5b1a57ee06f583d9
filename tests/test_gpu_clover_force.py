"""GPU tier of the clover force: b200_clover_force_accumulate against the numpy restatement (tests/clover_force_ref.py)
piece by piece and in total, in fp64 bit for bit against the host twin and between repeated calls; the pipeline
compute_clover_field -> asymmetric clover-PC Dirac -> invert_multishift_cg -> compute_clover_force against the restatement
fed the downloaded solutions, and against a finite difference of the action computed by the library alone; the refusals of
the operator-level call."""
import numpy as np
import pytest
import torch

import clover_build_ref as R
import clover_force_ref as CF
import oracle
from clover_force_cases import PIECES, TOL, Case, deviation, rotate_links, run
from force_twin import force_twin
from common import CudaMem, Problem
from quda_b200 import dirac as DR
from quda_b200 import dslash as D
from quda_b200 import fields as F
from quda_b200 import lib as L

pytestmark = pytest.mark.gpu

KAPPA, CSW = 0.12, 1.3
OFFSETS, COEFFS = [0.05, 0.2, 0.6], [0.5, 0.3, 0.2]
DEV = dict(to_dev=lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda(), to_host=lambda t: t.cpu().numpy(),
           ptr=lambda t: t.data_ptr())


@pytest.mark.parametrize("X", [(8, 8, 8, 8), (16, 16, 16, 16)])
@pytest.mark.parametrize("n", [1, 12])
@pytest.mark.parametrize("prec", [8, 4])
def test_library_matches_restatement_and_twin(X, n, prec):
    c = Case(X, n)
    lib = L.load()
    for piece in PIECES:
        got = run(lib, "b200", c, piece, prec, **DEV)
        assert deviation(got, c.reference(piece), c.mom) <= TOL[prec], piece
    again = run(lib, "b200", c, "all", prec, **DEV)
    assert np.array_equal(got, again)  # repeated calls: bit-identical
    if prec == 8:
        assert np.array_equal(got, run(force_twin(), "twin", c, "all", prec))


def _device_links(gauge, X):
    gbuf, gmeta = F.gauge_to_native(gauge, X, 8, 18)
    return D.GaugeField(CudaMem.put(gbuf), X, 8, 18, gmeta, t_boundary=-1)


def _solve(gauge, X, phi, matpc, U=None):
    """(solutions, tr log A per parity, operator) of the library's multi-shift CG on the asymmetric clover-PC operator"""
    U = U or _device_links(gauge, X)
    A, Ainv, trlog = D.compute_clover_field(gauge, X, 8, KAPPA, CSW)
    op = DR.Dirac("cloverpc", U, KAPPA, clover=A, clover_inv=Ainv, matpc_type=matpc)
    P = Problem(X, 8, 18, CudaMem)
    xs = [P.empty(1) for _ in OFFSETS]
    p = DR.invert_multishift_cg(op, None, xs, P.to_dev(phi), OFFSETS, tol=1e-12)
    assert max(p.true_res_offset[j] for j in range(len(OFFSETS))) < 1e-10
    return xs, trlog, op, P


@pytest.mark.parametrize("matpc", [DR.MATPC_EVEN_EVEN_ASYMMETRIC, DR.MATPC_ODD_ODD_ASYMMETRIC])
def test_pipeline_matches_restatement(matpc):
    X, dt, mult = (8, 8, 8, 8), 0.25, 2
    gauge = oracle.random_gauge(X, 8, seed=41, antiperiodic_t=True)
    phi = oracle.random_spinor(X, 8, seed=43) - 0.5
    xs, _, op, P = _solve(gauge, X, phi, matpc)
    rng = np.random.default_rng(3)
    V = int(np.prod(X))
    mom0 = 0.1 * CF.mom_from_matrices(CF.ta(rng.normal(size=(V, 4, 3, 3)) + 1j * rng.normal(size=(V, 4, 3, 3))))
    mom = torch.from_numpy(mom0).cuda()
    DR.compute_clover_force(mom, dt, xs, COEFFS, KAPPA, CSW, mult, gauge, op)
    want = CF.clover_force(mom0, dt, [P.to_host(x) for x in xs], COEFFS, -KAPPA ** 2, -CSW * KAPPA / 8, mult, gauge,
                           R.compute_clover(gauge, X, KAPPA * CSW), X, KAPPA, matpc)
    assert deviation(mom.cpu().numpy(), want, mom0) <= 1e-11


def test_finite_difference_through_the_library():
    """dS/d eps along U -> exp(eps H) U, with S = sum_i coeff_i phi^+ x_i - multiplicity tr log A_odd re-solved by the library
    at every point, against sum_links tr(H F), F = (mom_after - mom_before) / dt (the convention of
    test_twin_clover_force.py)"""
    X, dt, mult, matpc = (8, 8, 8, 8), 0.5, 1, DR.MATPC_EVEN_EVEN_ASYMMETRIC
    V = int(np.prod(X))
    gauge = oracle.random_gauge(X, 8, seed=47, antiperiodic_t=True)
    phi = oracle.random_spinor(X, 8, seed=49) - 0.5
    rng = np.random.default_rng(7)
    H = CF.ta(rng.normal(size=(4, V, 3, 3)) + 1j * rng.normal(size=(4, V, 3, 3)))
    xs, _, op, _ = _solve(gauge, X, phi, matpc)
    mom = torch.zeros((V, 4, 10), dtype=torch.float64, device="cuda")
    DR.compute_clover_force(mom, dt, xs, COEFFS, KAPPA, CSW, mult, gauge, op)
    predicted = np.einsum("mvij,vmji->", H, CF.mom_to_matrices(mom.cpu().numpy()) / dt).real

    def action(g):
        ys, trlog, _, P = _solve(g, X, phi, matpc)
        return sum(c * float(np.sum(phi * P.to_host(y))) for c, y in zip(COEFFS, ys)) - mult * trlog[1]

    eps = 1e-3
    S = {k: action(rotate_links(gauge, H, k * eps)) for k in (2, 1, -1, -2)}
    fd = (8 * (S[1] - S[-1]) - (S[2] - S[-2])) / (12 * eps)
    assert abs(fd - predicted) <= 1e-6 * abs(fd), (fd, predicted)


@pytest.mark.parametrize("kind", ["symmetric", "wilsonpc", "twistedmasspc", "partitioned"])
def test_operator_level_refusals(kind):
    X = (8, 8, 8, 8)
    P = Problem(X, 8, 18, CudaMem)
    A, Ainv, _ = D.compute_clover_field(P.gauge, X, 8, KAPPA, CSW)
    comm = None
    if kind == "partitioned":
        comm = L.Comm()
        comm.comm_dim[3] = 1
    if kind in ("symmetric", "partitioned"):
        matpc = DR.MATPC_EVEN_EVEN if kind == "symmetric" else DR.MATPC_EVEN_EVEN_ASYMMETRIC
        op = DR.Dirac("cloverpc", P.U, KAPPA, clover=A, clover_inv=Ainv, matpc_type=matpc, comm=comm)
    else:
        op = DR.Dirac(kind, P.U, KAPPA, matpc_type=DR.MATPC_EVEN_EVEN_ASYMMETRIC, mu=0.1)
    x = P.to_dev(P.spinor(seed=5))
    mom = torch.zeros((int(np.prod(X)), 4, 10), dtype=torch.float64, device="cuda")
    with pytest.raises(L.B200Error, match="error -1"):
        DR.compute_clover_force(mom, 0.1, [x], [1.0], KAPPA, CSW, 1, P.gauge, op)
    assert not mom.any()
