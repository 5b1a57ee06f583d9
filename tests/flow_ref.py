"""TEST ORACLE of the gradient flow and its observables, in numpy complex128.  The reference has no host code for either, so
this restates the formulas of include/kernels/gauge_wilson_flow.cuh (generator and RK3 of arXiv:1006.4518 App. C),
include/kernels/gauge_qcharge.cuh and lib/gauge_qcharge.cu (energy and charge from the clover F of
field_strength_tensor.cuh):
  Z_mu(x) = -TA(Omega_mu(x)),  Omega_mu(x) = U_mu(x) sum_i c_i path_i(x),  TA(M) = (M - M^+)/2 - tr(M - M^+)/6
  W1 = exp(Z0 / 4) W0,  W2 = exp(8/9 Z1 - 17/36 Z0) W1,  W3 = exp(3/4 Z2 - 8/9 Z1 + 17/36 Z0) W2,  Z_i = eps Z(W_i)
  E_spatial / E_temporal = sum over sites and planes (mu, nu) with mu < 3 / mu = 3 of -Re tr(Fhat^2), over V
  q(x) = -1/(4 pi^2) Re (tr F10 F32 - tr F20 F31 + tr F21 F30)
The exponential is the eigendecomposition of the Hermitian generator, independent of the library's closed form.  Fields:
QDP [4][V][3][3][2] parity-major outside, lexicographic complex inside (tests/clover_build_ref.py)."""
import numpy as np

import clover_build_ref as R
import clover_force_ref as CF
import gauge_cases as GC

PLANES = R.PLANES  # F10, F20, F21, F30, F31, F32


def expm(A):
    """exp(A) for anti-Hermitian A [..][3][3]: eigh of the Hermitian -i A"""
    w, v = np.linalg.eigh(-1j * A)
    return np.einsum("...ij,...j,...kj->...ik", v, np.exp(1j * w), v.conj())


def generator(U, paths, coeffs, sign=1.0):
    """Z[mu] = -TA(Omega_mu), lexicographic [4][t][z][y][x][3][3] (sign: a negative control flips it)"""
    return np.stack([-sign * CF.ta(U[mu] @ sum(c * GC.path_field(U, mu, p) for c, p in zip(coeffs, paths[mu])))
                     for mu in range(4)])


def rk3_step(U, paths, coeffs, eps):
    Z0 = eps * generator(U, paths, coeffs)
    W1 = expm(0.25 * Z0) @ U
    Z1 = eps * generator(W1, paths, coeffs)
    E2 = 8.0 / 9 * Z1 - 17.0 / 36 * Z0
    W2 = expm(E2) @ W1
    Z2 = eps * generator(W2, paths, coeffs)
    return expm(0.75 * Z2 - E2) @ W2


def euler_step(U, paths, coeffs, eps, sign=1.0):
    return expm(eps * generator(U, paths, coeffs, sign)) @ U


def flow(gauge, X, paths, coeffs, eps, n_steps, step=rk3_step):
    """QDP gauge after n_steps steps"""
    U = R.links(gauge, X)
    for _ in range(n_steps):
        U = step(U, paths, coeffs, eps)
    return GC.to_qdp(np.stack([R.from_lex(U[mu], X) for mu in range(4)]))


def field_strengths(gauge, X):
    U = R.links(gauge, X)
    return [R.field_strength(U, mu, nu) for mu, nu in PLANES]


def _re_tr(a, b):
    return np.einsum("...ij,...ji->...", a, b).real


def observables(gauge, X, pair_signs=(1, -1, 1)):
    """(energy (total, spatial, temporal), Q, q(x) parity-major); pair_signs: the signs of tr F0F5, tr F1F4, tr F2F3"""
    Fs = field_strengths(gauge, X)
    V = int(np.prod(X))
    e = [0.0, 0.0]
    for (mu, _), F in zip(PLANES, Fs):
        h = F - (np.trace(F, axis1=-2, axis2=-1) / 3)[..., None, None] * np.eye(3)
        e[mu == 3] -= _re_tr(h, h).sum() / V
    q = sum(s * _re_tr(Fs[i], Fs[5 - i]) for i, s in enumerate(pair_signs)) * (-1.0 / (4 * np.pi ** 2))
    q = R.from_lex(q, X)
    return (e[0] + e[1], e[0], e[1]), float(q.sum()), q


def action(gauge, X, paths, coeffs):
    """S = sum_i c_i sum_loops Re tr(1 - loop_i)"""
    return 3.0 * GC.loop_action(gauge, X, paths, coeffs, 1.0)


# ------------------------------------------------------------------ closed-form fields
def abelian_flux(X, planes):
    """links diag(e^{i theta}, e^{-i theta}, 1) with n flux quanta in each plane ((a, b), n) of `planes` (disjoint planes):
    every plaquette U_a(x) U_b(x+a) U_a(x+b)^+ U_b(x)^+ has the phase phi = 2 pi n / (L_a L_b), twisted at x_a = L_a - 1.
    Returns (QDP gauge, {(a, b): phi})."""
    t, z, y, x = np.meshgrid(*[np.arange(X[d]) for d in (3, 2, 1, 0)], indexing="ij")
    c = [x, y, z, t]
    theta = [np.zeros(c[0].shape) for _ in range(4)]
    phis = {}
    for (a, b), n in planes:
        phi = 2 * np.pi * n / (X[a] * X[b])
        phis[(a, b)] = phi
        theta[b] = theta[b] + phi * c[a]
        theta[a] = theta[a] - np.where(c[a] == X[a] - 1, phi * X[a] * c[b], 0.0)
    U = np.zeros((4,) + c[0].shape + (3, 3), dtype=np.complex128)
    for mu in range(4):
        U[mu, ..., 0, 0] = np.exp(1j * theta[mu])
        U[mu, ..., 1, 1] = np.exp(-1j * theta[mu])
        U[mu, ..., 2, 2] = 1.0
    return GC.to_qdp(np.stack([R.from_lex(U[mu], X) for mu in range(4)])), phis


# ------------------------------------------------------------------ symmetry maps
def random_su3(shape, seed):
    rng = np.random.default_rng(seed)
    z = (rng.normal(size=shape + (3, 3)) + 1j * rng.normal(size=shape + (3, 3))) / np.sqrt(2)
    q, r = np.linalg.qr(z)
    d = np.diagonal(r, axis1=-2, axis2=-1)
    q = q * (d / np.abs(d))[..., None, :]
    return q / np.linalg.det(q)[..., None, None] ** (1.0 / 3)


def gauge_transform(gauge, X, g):
    """U_mu(x) -> g(x) U_mu(x) g(x + mu)^+, g lexicographic [t][z][y][x][3][3]"""
    U = R.links(gauge, X)
    out = [g @ U[mu] @ R.dag(R.shift(g, mu, 1)) for mu in range(4)]
    return GC.to_qdp(np.stack([R.from_lex(u, X) for u in out]))


def reflect_x(gauge, X):
    """x_0 -> -x_0: U'_0(x) = U_0(Rx - 0)^+, U'_nu(x) = U_nu(Rx)"""
    U = R.links(gauge, X)

    def refl(a):
        return np.roll(np.flip(a, axis=3), 1, axis=3)  # a(-x_0)

    out = [R.dag(refl(R.shift(U[0], 0, -1)))] + [refl(U[mu]) for mu in range(1, 4)]
    return GC.to_qdp(np.stack([R.from_lex(u, X) for u in out]))
