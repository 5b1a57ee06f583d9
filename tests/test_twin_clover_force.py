"""CPU tier of the clover force: the numpy restatement (tests/clover_force_ref.py) pinned by a finite difference of the action
and by gauge covariance; the host twin of b200_clover_force_accumulate (the library's site code built for the CPU by
tests/forcetwin) against the restatement, piece by piece and in total; the twin's argument checks."""
import ctypes as C

import numpy as np
import pytest
import scipy.linalg as sl

import clover_build_ref as R
import clover_force_ref as CF
import oracle
from clover_force_cases import PIECES, TOL, Case, deviation, rotate_links, run
from force_twin import force_twin
from quda_b200 import lib as L

KAPPA, CSW = 0.12, 1.3
SHIFTS, COEFFS = [0.1, 0.3, 1.0], [0.7, 0.2, 0.1]


# ------------------------------------------------------------------ finite difference
# Convention (the reference's integrator, under which it conserves H): momentum action sum -1/2 tr P^2
# (include/kernels/momentum.cuh:29-50) and gauge update U <- exp(dt P) U (include/kernels/gauge_update.cuh).  Then
# dP/dt = TA(F) where dS/d eps [U -> exp(eps H) U] = sum_links tr(H F), so F = (mom_after - mom_before) / dt must satisfy that
# identity for the action S the force belongs to.  That action is
#   S(U) = sum_i coeff_i phi^+ (Mhat^+ Mhat + sigma_i)^-1 phi - c multiplicity tr log A_other(U),   c = 1:
# with asymmetric preconditioning det M = det A_other det Mhat, so the 2-flavour weight det(M^+ M) = det(A_other)^2
# det(Mhat^+ Mhat) puts -2 tr log A_other beside the pseudofermion of (Mhat^+ Mhat)^-1, and the reference's multiplicity
# (sigma_coeff = 2 ck multiplicity dt against the pseudofermion's 2 ck coeff dt) counts those tr log A_other terms.
C_TRLOG = 1.0


def _action(gauge, X, phi, coeffs, matpc, csw):
    """(S, solutions x_i as DeGrand-Rossi host spinors, packed A); Mhat is the oracle's asymmetric clover matpc, the shifted
    normal systems are solved densely"""
    A = R.compute_clover(gauge, X, KAPPA * csw)
    Ainv = oracle.clover_invert(A)
    Vh = int(np.prod(X)) // 2
    n = 12 * Vh
    M = np.zeros((n, n), dtype=complex)
    e = np.zeros((Vh, 4, 3, 2))
    for k in range(n):
        e[:] = 0
        e.reshape(-1, 2)[k, 0] = 1.0
        o = oracle.clover_matpc(gauge, A, Ainv, e, X, KAPPA, matpc, 0)
        M[:, k] = (o[..., 0] + 1j * o[..., 1]).ravel()
    N = M.conj().T @ M
    ph = (phi[..., 0] + 1j * phi[..., 1]).ravel()
    sols = [sl.solve(N + s * np.eye(n), ph, assume_a="pos") for s in SHIFTS]
    S = sum(c * np.vdot(ph, y).real for c, y in zip(coeffs, sols))
    par = 0 if matpc == oracle.MATPC_EVEN_EVEN_ASYM else 1
    xs = [np.stack([y.reshape(Vh, 4, 3).real, y.reshape(Vh, 4, 3).imag], -1) for y in sols]
    return S, R.trlog(A)[1 - par], xs, A


@pytest.mark.parametrize("case,matpc,antiperiodic,mult", [
    ("hop", oracle.MATPC_EVEN_EVEN_ASYM, True, 1),
    ("det", oracle.MATPC_EVEN_EVEN_ASYM, False, 2),
    ("all", oracle.MATPC_EVEN_EVEN_ASYM, False, 1),
    ("all", oracle.MATPC_ODD_ODD_ASYM, True, 2)])
def test_finite_difference_pins_the_restatement(case, matpc, antiperiodic, mult):
    """hopping only (c_sw = 0), determinant only (coeff = 0) and everything, so that no relative factor between the terms
    can hide in the total"""
    X = (4, 4, 4, 4)
    V = int(np.prod(X))
    csw = 0.0 if case == "hop" else CSW
    coeffs = [0.0] * 3 if case == "det" else COEFFS
    gauge = oracle.random_gauge(X, 8, seed=3, antiperiodic_t=antiperiodic)
    phi = oracle.random_spinor(X, 8, seed=9) - 0.5
    rng = np.random.default_rng(1)
    H = CF.ta(rng.normal(size=(4, V, 3, 3)) + 1j * rng.normal(size=(4, V, 3, 3)))
    _, _, xs, A = _action(gauge, X, phi, coeffs, matpc, csw)
    dt = 0.3
    mom0 = CF.mom_from_matrices(CF.ta(rng.normal(size=(V, 4, 3, 3)) + 0j))
    mom1 = CF.clover_force(mom0, dt, xs, coeffs, -KAPPA ** 2, -csw * KAPPA / 8, mult, gauge, A, X, KAPPA, matpc)
    Fm = CF.mom_to_matrices(mom1 - mom0) / dt  # [V][4][3][3]
    predicted = np.einsum("mvij,vmji->", H, Fm).real
    eps, S = 1e-4, {}
    for k in (2, 1, -1, -2):  # fourth-order central difference
        s, tl, _, _ = _action(rotate_links(gauge, H, k * eps), X, phi, coeffs, matpc, csw)
        S[k] = s - C_TRLOG * mult * tl
    fd = (8 * (S[1] - S[-1]) - (S[2] - S[-2])) / (12 * eps)
    assert abs(fd - predicted) <= 1e-7 * abs(fd), (fd, predicted)


def test_gauge_covariance():
    """F(U^g) = g F(U) g^+ site by site, with the spinors rotated along (x -> g x)"""
    X = (4, 4, 4, 4)
    c = Case(X, 2)
    rng = np.random.default_rng(5)
    V = int(np.prod(X))
    qm, r = np.linalg.qr(rng.normal(size=(V, 3, 3)) + 1j * rng.normal(size=(V, 3, 3)))
    g = qm * (np.diagonal(r, axis1=1, axis2=2) / np.abs(np.diagonal(r, axis1=1, axis2=2)))[:, None, :]
    g = g / np.linalg.det(g)[:, None, None] ** (1.0 / 3.0)
    g_lex = R.to_lex(g, X)
    U = c.gauge[..., 0] + 1j * c.gauge[..., 1]
    Ug = np.stack([R.from_lex(g_lex @ R.to_lex(U[mu], X) @ R.dag(R.shift(g_lex, mu, 1)), X) for mu in range(4)])
    gauge_g = np.stack([Ug.real, Ug.imag], -1)
    packed_g = R.compute_clover(gauge_g, X, 0.12 * 1.3)
    fc, eps, sc = c.coefficients("all")
    zero = np.zeros_like(c.mom)
    lex = [CF.host_to_lex(v, X) for v in c.xs], [CF.host_to_lex(v, X) for v in c.ps]
    rot = lambda f: np.einsum("...ab,...sb->...sa", g_lex, f)  # noqa: E731
    f0 = CF.mom_to_matrices(CF.accumulate(zero, c.gauge, c.packed, *lex, fc, eps, sc, 1, X))
    f1 = CF.mom_to_matrices(CF.accumulate(zero, gauge_g, packed_g, [rot(v) for v in lex[0]], [rot(v) for v in lex[1]], fc,
                                          eps, sc, 1, X))
    want = g[:, None] @ f0 @ R.dag(g)[:, None]
    assert np.abs(f1 - want).max() <= 1e-12 * np.abs(f0).max()


# ------------------------------------------------------------------ the twin against the restatement
@pytest.mark.parametrize("X", [(4, 4, 4, 4), (8, 8, 8, 8)])
@pytest.mark.parametrize("n", [1, 12])
@pytest.mark.parametrize("prec", [8, 4])
def test_twin_matches_restatement(X, n, prec):
    c = Case(X, n)
    for piece in PIECES:
        got = run(force_twin(), "twin", c, piece, prec)
        dev = deviation(got, c.reference(piece), c.mom)
        assert dev <= TOL[prec], (piece, dev)


def test_twin_is_deterministic():
    c = Case((4, 4, 4, 4), 3)
    assert np.array_equal(run(force_twin(), "twin", c, "all", 8), run(force_twin(), "twin", c, "all", 8))


@pytest.mark.parametrize("case", ["n_0", "n_33", "odd_X", "null_mom", "null_link", "null_x", "null_packed", "prec_2",
                                  "trlog_parity_2", "coeff_nan", "eps_inf", "sigma_nan"])
def test_accumulate_refuses(case):
    lib = force_twin()
    buf = np.zeros(64)
    p = buf.ctypes.data
    n, prec, tp, sc = 2, 8, 1, 0.1
    X = (C.c_int * 4)(4, 4, 4, 4)
    q = (C.c_void_p * 4)(p, p, p, p)
    xs = (C.c_void_p * 40)(*([p] * 40))
    fc = (C.c_double * 40)(*([0.1] * 40))
    eps = (C.c_double * 80)(*([0.1] * 80))
    mom, packed = p, p
    if case == "n_0":
        n = 0
    elif case == "n_33":
        n = 33
    elif case == "odd_X":
        X[2] = 5
    elif case == "null_mom":
        mom = None
    elif case == "null_link":
        q[3] = None
    elif case == "null_x":
        xs[1] = None
    elif case == "null_packed":
        packed = None
    elif case == "prec_2":
        prec = 2
    elif case == "trlog_parity_2":
        tp = 2
    elif case == "coeff_nan":
        fc[1] = float("nan")
    elif case == "eps_inf":
        eps[3] = float("inf")
    else:
        sc = float("nan")
    assert lib.twin_clover_force_accumulate(mom, q, packed, X, prec, n, xs, xs, fc, eps, sc, tp, None) == -1  # B200_ERR_INVALID
    assert b"b200_clover_force_accumulate" in lib.twin_last_error()
