"""TEST ORACLE of gauge smearing, in numpy complex128, written from the definitions (not from the reference's index
arithmetic).  S_mu(x) is the sum of the staples of U_mu(x) in the smeared planes (mu, nu), nu != mu and nu != the
ignored direction, a staple being
  A_nu(x) B_mu(x + nu) A_nu(x + mu)^+ + A_nu(x - nu)^+ B_mu(x - nu) A_nu(x - nu + mu)
with the mu-links from the field B and the nu-links from A; d is the number of smeared directions.
  APE     U' = P[(1 - alpha) 1 + alpha / (2 (d - 1)) S U^+] U
  stout   U' = exp(rho TA(S U^+)) U,  TA(M) = (M - M^+)/2 - tr(M - M^+)/6
  over-improved stout (Moran & Leinweber, arXiv:0801.1165): rho TA(((5 - 2 eps)/3 S - (1 - eps)/12 R) U^+), R the 2x1
          rectangle staples, taken here as the adjoints of the closed 2x1 loops through U_mu(x)
  HYP     (Hasenfratz & Knechtli, hep-lat/0103029) 4-d:
            Vbar_{mu;nu rho} = P[(1 - a3) + a3/2 sum_{eta != mu,nu,rho} staple(U, U) U^+] U
            Vtil_{mu;nu}     = P[(1 - a2) + a2/4 sum_{rho != mu,nu} staple(mu-links Vbar_{mu;rho nu}, rho-links Vbar_{rho;nu mu}) U^+] U
            V_mu             = P[(1 - a1) + a1/6 sum_{nu != mu} staple(mu-links Vtil_{mu;nu}, nu-links Vtil_{nu;mu}) U^+] U
          3-d (one direction ignored): Vbar_{mu;nu} from the one remaining plane, then the last level with a2/4 on
          (Vbar_{mu;nu}, Vbar_{nu;mu})
P is the unitary polar factor (SVD) divided by the principal cube root of its determinant, arg in (-pi, pi]; the
exponential is an eigendecomposition (flow_ref.expm).  Fields: QDP [4][V][3][3][2] outside, lexicographic complex inside."""
import numpy as np

import clover_build_ref as R
import clover_force_ref as CF
import flow_ref as FR
import gauge_cases as GC


def principal_arg(z):
    a = np.angle(z)
    return np.where(a <= -np.pi, np.pi, a)


def project(W):
    """SU(3) projection of [..][3][3]: the polar factor u vh of the SVD over the principal cube root of its determinant"""
    u, _, vh = np.linalg.svd(W)
    P = u @ vh
    det = np.linalg.det(P)
    return P * (np.exp(-1j * principal_arg(det) / 3) / np.abs(det) ** (1.0 / 3))[..., None, None]


def staple(B, A, mu, nu):
    """the two staples of the link mu in the plane (mu, nu), mu-links from B, nu-links from A"""
    Am = R.shift(A, nu, -1)
    return A @ R.shift(B, nu, 1) @ R.dag(R.shift(A, mu, 1)) + R.dag(Am) @ R.shift(B, nu, -1) @ R.shift(Am, mu, 1)


def level(U, S, alpha, c, sum_projection=False):
    """P[(1 - alpha) 1 + c S U^+] U; sum_projection: the negative control P[(1 - alpha) U + c S]"""
    if sum_projection:
        return project((1 - alpha) * U + c * S)
    return project((1 - alpha) * np.eye(3) + c * S @ R.dag(U)) @ U


def _rect_loops(mu, nu):
    return [l for l in GC.rectangle_loops(mu) if any(abs(s) == nu + 1 for s in l)]


def _loop(U, mu, loop):
    return U[mu] @ GC.path_field(U, mu, [GC._enc(s) for s in loop[1:]])


def _step(U, kind, dirs, c, control):
    out = U.copy()
    d = len(dirs)
    if kind == "ape":
        norm = control.get("ape_norm", 2 * (d - 1))
        for mu in dirs:
            S = sum(staple(U[mu], U[nu], mu, nu) for nu in dirs if nu != mu)
            out[mu] = level(U[mu], S, c["alpha"], c["alpha"] / norm, control.get("sum_projection", False))
    elif kind in ("stout", "ovrimp_stout"):
        eps = c.get("epsilon", 0.0)
        cp, cr = ((5 - 2 * eps) / 3, (1 - eps) / 12) if kind == "ovrimp_stout" else (1.0, 0.0)
        for mu in dirs:
            M = sum(staple(U[mu], U[nu], mu, nu) for nu in dirs if nu != mu) @ R.dag(U[mu]) * cp
            if cr:
                M = M - cr * sum(R.dag(_loop(U, mu, l)) for nu in dirs if nu != mu for l in _rect_loops(mu, nu))
            out[mu] = FR.expm(c["rho"] * CF.ta(M)) @ U[mu]
    elif kind == "hyp" and d == 4:
        a1, a2, a3 = c["alpha1"], c["alpha2"], c["alpha3"]
        vbar = {}
        for mu in dirs:
            for nu in dirs:
                for rho in dirs:
                    if len({mu, nu, rho}) == 3:
                        (eta,) = set(dirs) - {mu, nu, rho}
                        vbar[mu, frozenset((nu, rho))] = level(U[mu], staple(U[mu], U[eta], mu, eta), a3, a3 / 2)
        vtil = {}
        for mu in dirs:
            for nu in dirs:
                if nu == mu:
                    continue
                rhos = [r for r in dirs if r not in (mu, nu)]
                if control.get("wrong_level2"):  # the mu-links decorated in the wrong plane
                    S = sum(staple(vbar[mu, frozenset((nu, 6 - mu - nu - r))], vbar[r, frozenset((nu, mu))], mu, r) for r in rhos)
                else:
                    S = sum(staple(vbar[mu, frozenset((r, nu))], vbar[r, frozenset((nu, mu))], mu, r) for r in rhos)
                vtil[mu, nu] = level(U[mu], S, a2, a2 / 4)
        for mu in dirs:
            S = sum(staple(vtil[mu, nu], vtil[nu, mu], mu, nu) for nu in dirs if nu != mu)
            out[mu] = level(U[mu], S, a1, a1 / 6)
    else:  # 3-d HYP
        a2, a3 = c["alpha2"], c["alpha3"]
        vbar = {}
        for mu in dirs:
            for nu in dirs:
                if nu != mu:
                    (eta,) = set(dirs) - {mu, nu}
                    vbar[mu, nu] = level(U[mu], staple(U[mu], U[eta], mu, eta), a3, a3 / 2)
        for mu in dirs:
            S = sum(staple(vbar[mu, nu], vbar[nu, mu], mu, nu) for nu in dirs if nu != mu)
            out[mu] = level(U[mu], S, a2, a2 / 4)
    return out


def smear(gauge, X, kind, n_steps, dir_ignore=-1, control=None, **coeffs):
    """QDP gauge after n_steps steps of `kind`; dir_ignore in 0..3 leaves that direction out (-1 or 4: none)"""
    dirs = [d for d in range(4) if d != dir_ignore]
    U = R.links(gauge, X)
    for _ in range(n_steps):
        U = _step(U, kind, dirs, coeffs, control or {})
    return GC.to_qdp(np.stack([R.from_lex(U[mu], X) for mu in range(4)]))
