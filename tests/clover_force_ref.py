"""TEST ORACLE of the clover fermion force, in numpy complex128: the momentum update of computeCloverForceQuda for the
non-twisted Wilson-clover operator with asymmetric even-odd preconditioning.  Restated from the formulas of the reference's
lib/clover_force.cpp:11-104 (preparation of p, order of the pieces), include/kernels/clover_outer_product.cuh (hopping
force), clover_sigma_outer_product.cuh (sigma outer product), clover_trace.cuh (tr[sigma A^-1] from the chiral blocks),
clover_deriv.cuh (insertion into the leaves) and momentum.cuh (updateMomentum: mom -= TA(force)).  The reference's own
host implementation needs Eigen and working ColorSpinorField objects, so this restatement is pinned instead by a finite
difference of the action (tests/test_twin_clover_force.py).

Field orders: spinors are complex [..., 4 spins, 3 colours] in the UKQCD basis (the native basis; fields.rotate_basis
converts the DeGrand-Rossi host order), links and oprod complex [..][3][3]; mom [V][4][10] reals (the (01), (02), (12)
complex entries, the three imaginary diagonals, one pad).  Internally every field is lexicographic [t][z][y][x] as in
tests/clover_build_ref.py, whose helpers this module uses."""
import numpy as np

import oracle
from clover_build_ref import PLANES, dag, from_lex, invert, links, shift, to_lex, unpack
from quda_b200 import fields as F

_i = 1j
# gamma_mu in the UKQCD basis, read off core.h's project(): P(mu, s) = 1 + s gamma_mu
GAMMA = [np.array([[0, 0, 0, _i], [0, 0, _i, 0], [0, -_i, 0, 0], [-_i, 0, 0, 0]]),
         np.array([[0, 0, 0, 1], [0, 0, -1, 0], [0, -1, 0, 0], [1, 0, 0, 0]]),
         np.array([[0, 0, _i, 0], [0, 0, 0, -_i], [-_i, 0, 0, 0], [0, _i, 0, 0]]),
         np.diag([1, 1, -1, -1]).astype(complex)]
GAMMA5_DR = np.array([1.0, 1.0, -1.0, -1.0])  # gamma_5 of the DeGrand-Rossi host basis (diagonal)
OD = [(0, 1), (0, 2), (1, 2)]


def sigma(a, b):
    """the reference's ColorSpinor::sigma(a, b) = gamma_a gamma_b (a != b)"""
    return GAMMA[a] @ GAMMA[b]


def spin(m, v):
    """m (4x4) applied to the spin index of v [..., 4, 3]"""
    return np.einsum("st,...tc->...sc", m, v)


def outer(a, b):
    """tr_spin[a b^+]: (j, k) = sum_s a(s, j) conj(b(s, k))"""
    return np.einsum("...sj,...sk->...jk", a, np.conj(b))


def parity_lex(X):
    t, z, y, x = np.meshgrid(*[np.arange(X[d]) for d in (3, 2, 1, 0)], indexing="ij")
    return (x + y + z + t) & 1


# ------------------------------------------------------------------ field conversions
def host_to_lex(host, X):
    """DeGrand-Rossi host spinor [V parity-major][4][3][2] -> complex UKQCD [t][z][y][x][4][3]"""
    v = F.rotate_basis(host, True)
    return to_lex(v[..., 0] + 1j * v[..., 1], X)


def ta(m):
    """traceless anti-Hermitian part"""
    a = 0.5 * (m - dag(m))
    tr = np.trace(a, axis1=-2, axis2=-1).imag / 3.0
    return a - 1j * tr[..., None, None] * np.eye(3)


def mom_from_matrices(m):
    """[...][3][3] traceless anti-Hermitian -> [...][10]"""
    out = np.zeros(m.shape[:-2] + (10,))
    for n, (i, j) in enumerate(OD):
        out[..., 2 * n], out[..., 2 * n + 1] = m[..., i, j].real, m[..., i, j].imag
    for k in range(3):
        out[..., 6 + k] = m[..., k, k].imag
    return out


def mom_to_matrices(mom):
    """[...][10] -> [...][3][3] anti-Hermitian"""
    mom = np.asarray(mom, dtype=np.float64)
    m = np.zeros(mom.shape[:-1] + (3, 3), dtype=np.complex128)
    for n, (i, j) in enumerate(OD):
        m[..., i, j] = mom[..., 2 * n] + 1j * mom[..., 2 * n + 1]
        m[..., j, i] = -np.conj(m[..., i, j])
    for k in range(3):
        m[..., k, k] = 1j * mom[..., 6 + k]
    return m


# ------------------------------------------------------------------ the three pieces
def hop_force(U, xs, ps, force_coeff):
    """[4][lex][3][3]: U_mu(x) sum_i c_i tr_spin[(1+g_mu) x_i(x+mu) p_i(x)^+ + (1-g_mu) p_i(x+mu) x_i(x)^+]"""
    out = []
    one = np.eye(4)
    for mu in range(4):
        r = 0
        for x, p, c in zip(xs, ps, force_coeff):
            r = r + c * outer(spin(one + GAMMA[mu], shift(x, mu, 1)), p)
            r = r + c * outer(spin(one - GAMMA[mu], shift(p, mu, 1)), x)
        out.append(U[mu] @ r)
    return np.stack(out)


def sigma_oprod(xs, ps, eps, X):
    """[6][lex][3][3]: R - R^+, R = sum_i eps_i[parity(x)] tr_spin[sigma(nu, mu) x_i p_i^+] for plane (mu, nu)"""
    par = parity_lex(X)
    out = []
    for mu, nu in PLANES:
        r = 0
        for x, p, e in zip(xs, ps, eps):
            w = np.where(par == 0, e[0], e[1])[..., None, None]
            r = r + w * outer(spin(sigma(nu, mu), x), p)
        out.append(r - dag(r))
    return np.stack(out)


def sigma_trace(packed, coeff, parity, X):
    """[6][lex][3][3]: coeff tr_spin[sigma A^-1] on the sites of `parity` (zero elsewhere), written from the chiral blocks of
    A^-1 as clover_trace.cuh does (A0, A1: the two 6x6 blocks; UL, LR, UR, LL their 3x3 quadrants)"""
    inv = invert(np.asarray(packed, dtype=np.float64))[0]
    H = unpack(inv)  # [V][2][6][6]
    UL, LR, UR, LL = H[..., :3, :3], H[..., 3:, 3:], H[..., :3, 3:], H[..., 3:, :3]
    I = 1j
    mats = [I * (LR[:, 0] + LR[:, 1] - UL[:, 0] - UL[:, 1]),   # (1, 0)
            UR[:, 0] - LL[:, 0] + UR[:, 1] - LL[:, 1],          # (2, 0)
            -I * (UR[:, 0] + LL[:, 0] + UR[:, 1] + LL[:, 1]),   # (2, 1)
            I * (UR[:, 0] + LL[:, 0] - UR[:, 1] - LL[:, 1]),    # (3, 0)
            UR[:, 0] - LL[:, 0] - UR[:, 1] + LL[:, 1],          # (3, 1)
            I * (UL[:, 0] - LR[:, 0] - UL[:, 1] + LR[:, 1])]    # (3, 2)
    mask = (parity_lex(X) == parity)[..., None, None]
    return np.stack([np.where(mask, coeff * to_lex(m, X), 0) for m in mats])


def deriv(U, O):
    """[4][lex][3][3]: the insertion of oprod O[6] at the corners of the upper leaf U_mu(x) U_nu(x+mu) U_mu(x+nu)^+ U_nu(x)^+
    and the lower leaf U_nu(x-nu)^+ U_mu(x-nu) U_nu(x+mu-nu) U_mu(x)^+, summed over nu != mu (clover_deriv.cuh)"""
    out = []
    for mu in range(4):
        f = 0
        for nu in range(4):
            if nu == mu:
                continue
            t = PLANES.index((max(mu, nu), min(mu, nu)))
            Ot = O[t]
            s = lambda a, dm, dn: shift(shift(a, mu, dm), nu, dn)  # noqa: E731  a(x + dm mu + dn nu)
            U1, U2, U3, U4 = U[mu], s(U[nu], 1, 0), s(U[mu], 0, 1), U[nu]
            up = (U1 @ U2 @ dag(U3) @ dag(U4) @ Ot + U1 @ U2 @ s(Ot, 1, 1) @ dag(U3) @ dag(U4)
                  + U1 @ U2 @ dag(U3) @ s(Ot, 0, 1) @ dag(U4) + U1 @ s(Ot, 1, 0) @ U2 @ dag(U3) @ dag(U4))
            L1, L2, L3, L4 = s(U[nu], 0, -1), s(U[mu], 0, -1), s(U[nu], 1, -1), U[mu]
            lo = (dag(L1) @ L2 @ s(Ot, 1, -1) @ L3 @ dag(L4) + Ot @ dag(L1) @ L2 @ L3 @ dag(L4)
                  + dag(L1) @ L2 @ L3 @ s(Ot, 1, 0) @ dag(L4) + dag(L1) @ s(Ot, 0, -1) @ L2 @ L3 @ dag(L4))
            sg = -1.0 if nu < mu else 1.0
            f = f + sg * up - sg * lo
        out.append(f)
    return np.stack(out)


def accumulate(mom, gauge, packed, xs, ps, force_coeff, eps, sigma_coeff, trlog_parity, X):
    """b200_clover_force_accumulate: mom [V][4][10] after the update.  xs, ps: lists of full-lattice UKQCD lexicographic
    spinors; eps[i] = (even sites, odd sites)."""
    U = links(gauge, X)
    O = sigma_oprod(xs, ps, eps, X) + sigma_trace(packed, sigma_coeff, trlog_parity, X)
    f = hop_force(U, xs, ps, force_coeff) + deriv(U, O)
    m = mom_to_matrices(mom) - np.stack([from_lex(ta(f[mu]), X) for mu in range(4)], axis=1)
    return mom_from_matrices(ta(m))


# ------------------------------------------------------------------ operator level
def prepare(gauge, packed, x, X, kappa, matpc):
    """(x_full, p_full) as DeGrand-Rossi host spinors [V][4][3][2] from the solution x [Vh][4][3][2] on the matpc parity:
    lib/clover_force.cpp:46-80 along its dagger branch (the dagger Dslash and M-dagger first, then the plain Dslash), with
    the oracle's operators.  For solutions of (Mhat^+ Mhat + sigma) x = phi this is the derivative of phi^+ (Mhat^+ Mhat +
    sigma)^-1 phi; the reference's non-dagger branch would give that of the Mhat Mhat^+ action instead."""
    par = 0 if matpc == oracle.MATPC_EVEN_EVEN_ASYM else 1
    oth = 1 - par
    A = np.asarray(packed, dtype=np.float64)
    Ainv = oracle.clover_invert(A)
    g5 = lambda v: v * GAMMA5_DR[:, None, None]  # noqa: E731
    x = np.asarray(x, dtype=np.float64)
    t = g5(x)
    x_oth = oracle.apply_clover(Ainv, oracle.wil_dslash(gauge, t, X, oth, 1), X, oth)  # dagger Dslash: A^-1 D^+
    p_par = oracle.clover_matpc(gauge, A, Ainv, t, X, kappa, matpc, 1)  # Mhat^+
    x_oth = g5(x_oth)
    p_oth = oracle.apply_clover(Ainv, oracle.wil_dslash(gauge, p_par, X, oth, 0), X, oth)
    halves = lambda a, b: np.concatenate([a, b] if par == 0 else [b, a])  # noqa: E731
    return halves(x, x_oth), halves(g5(p_par), g5(p_oth))


def coefficients(dt, coeffs, kappa2, ck, multiplicity, matpc):
    """force_coeff, eps (per site parity), sigma_coeff and the tr log parity of computeCloverForceQuda
    (lib/interface_quda.cpp:4585-4609).  eps = (this parity, other parity) of the matpc."""
    par = 0 if matpc == oracle.MATPC_EVEN_EVEN_ASYM else 1
    fc = [2.0 * dt * c * kappa2 for c in coeffs]
    eps = []
    for c in coeffs:
        e = (2.0 * ck * c * dt, -kappa2 * 2.0 * ck * c * dt)
        eps.append(e if par == 0 else e[::-1])
    return fc, eps, 2.0 * ck * multiplicity * dt, 1 - par


def clover_force(mom, dt, xs, coeffs, kappa2, ck, multiplicity, gauge, packed, X, kappa, matpc):
    """computeCloverForceQuda: mom [V][4][10] after the update, from the single-parity DeGrand-Rossi solutions xs"""
    xf, pf = [], []
    for x in xs:  # the dagger branch passes p in x's place and x in p's (lib/clover_force.cpp:84-98)
        a, b = prepare(gauge, packed, x, X, kappa, matpc)
        xf.append(host_to_lex(b, X))
        pf.append(host_to_lex(a, X))
    fc, eps, sc, tp = coefficients(dt, coeffs, kappa2, ck, multiplicity, matpc)
    return accumulate(mom, gauge, packed, xf, pf, fc, eps, sc, tp, X)
