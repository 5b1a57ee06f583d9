"""High-precision reference of the gauge half of an HMC step with a per-element bound on the kernels' rounding error
(test-only, numpy).  The companion of tests/precise.py and tests/precise_clover.py for the kernels of gauge.h:
gauge_force_kernel, gauge_update_kernel (exact and order-8), mom_action_kernel and plaquette_kernel.

The flat checks of tests/test_twin_gauge.py divide the force error by the largest force of the whole field, let the update
error grow with |dt P|^2 and compare the fp32 momentum action with 1e-7 sum |m|.  Here every element is checked against
its own bound.  The reference reads exactly the values the kernel reads (links and momenta rounded to the field's
precision, (T)coeff, (T)eb3, (T)dt) and computes in long double for fp64 kernels and in float64 for fp32 kernels.  Every
real output must satisfy

    |got - ref| <= sqrt2 gamma_K u T + E_in + u_P |ref|

with the notation of precise_clover.py: gamma_K = K u / (1 - K u), T the same computation on absolute values (complex
moduli), E_in a propagated error of an earlier stage and u_P |ref| the output rounding (precise.out_bound).  The counts
are read off gauge.h (a 3x3 complex product, su3_mul_op, is a chain of 6 fmas per real output: 6 roundings):

* Force (gauge_force_site).  Path i of L_i links: the L_i - 1 chained su3_mul_op products (6 (L_i - 1)); the
  accumulation s = fma_rn(c_i, m, s) over the paths, in which path i (from 0) sees n - i roundings; f = U_mu(x) s (6);
  eb3 * f (1).  So path i carries K_i = 6 (L_i - 1) + (n - i) + 7 and the bound of f is sqrt2 |eb3| |U_mu| sum_i
  gamma_{K_i} |c_i| |path_i|.  mom_sub_ta (clover_force.h) then maps the error of f linearly: an off-diagonal component
  takes (E_ij + E_ji) / 2, a diagonal one 2/3 E_kk + 1/3 of the other two (the trace it subtracts cancels exactly);
  its own roundings are precise_clover.K_TA = 9 on |mom| + 2 |f|.  The pad mom[9] is never written.
* Exact update (su3_exp, su3_exp_coeffs): exp(A) U, A = dt P, in four parts.
  1. The rounding of A: the trace removal of mom_traceless ((m6 + m7 + m8) / 3: 3 roundings, m - tr: 1) and dt * p (1).
     It enters with weight <= 1: the Frechet derivative of exp at an anti-Hermitian A is E -> int_0^1 e^{sA} E
     e^{(1-s)A} ds, whose 2-norm is <= ||E||_2 because e^{sA} is unitary; so the 2-norm of the error of exp(A) U is <=
     ||dA||_F ||U||_2, which bounds every element.
  2. The invariants in T: Q^2 (6), c1 = tr Q^2 / 2 (2 adds; * 0.5 is exact): `K_C1` = 8 on tr |Q| |Q| / 2;
     t3 = Re tr(Q Q^2) as a chain of 18 fmas on top of Q^2's 6, then / 3: `K_C0` = 25 on sum |Q| |Q|^2 / 3.  They move
     F = f0 + f1 Q + f2 Q^2 by |dF/dc0| dc0 + |dF/dc1| dc1, the derivatives taken by differences of the long-double
     closed form (one-sided where c0 + h would pass c0_max, where su3_exp_coeffs clamps r), times 2; below c1 = 1e-3
     |dF/dc_k| <= 1 elementwise (the Taylor coefficients: dF/dc1 ~ -1/2 + i Q / 6 + Q^2 / 24, dF/dc0 ~ i / 6 + ...).
  3. su3_exp_coeffs in double, by a running error analysis of its own operations (precise._add / _mul / _cmul: every
     operation adds u (|value| + error)): sqrt(c1 / 3), r and its clamp, the Newton solve for cos(theta / 3) (its
     derivative 12 c^2 - 3 >= 6 on [cos(pi/6), 1], so |dc| <= |dr| / 6 + `NEWTON_U` u), w^2 = c1 (1 - c^2) (w enters
     only through the even cos w and sin w / w, whose derivatives in w^2 are <= 1/2 and 1/6), sin w / w, the h_j of
     M&P eqs. 30-32 on their values and errors, den = 9 u^2 - w^2 and h_j / den.  sincos_rn's error is its
     argument's error plus `SINCOS_U` u absolute: the Cody-Waite reduction (x - k pio2_1 exact for |k| < 2^20, one rounding of the pio2_1t term, pi/2 - pio2_1 -
     pio2_1t < 2.1e-21 per unit of k) and fdlibm's kernels on [-pi/4, pi/4] (< 1 ulp each, here with fma chains).
     The series branch (c1 < kExpSeriesC1) adds its truncation ||Q||_2^6 / 720 e^{||Q||_2} and 3 roundings of each
     coefficient.  In fp32 the coefficients are rounded to float (u_f |f_j|).
  4. The assembly f0 + f1 Q + f2 Q^2 in T (5 roundings on top of Q^2's 6) and the product with U (6): `K_ASM` = 17
     on (|f0| + |f1| |Q| + |f2| |Q|^2) |U|; parts 2 and 3 reach the output through |U|.
* Order-8 update: the reference is the same Horner polynomial r <- U + (dt / k) P r, k = kUpdateOrder .. 1, in long
  double, so the bound is rounding only: per step, sc = dt / k (1), sc * p (1), P's trace removal (as part 1 above)
  and su3_mul_op with accumulation onto U (6), propagated through |sc P| as a running bound.
* Momentum action (mom_action_site): per link 6 fmas for the off-diagonal squares, fma(0.5, dg, off) and - 4 (2), four
  links into s (4): 12; a 128-leaf CTA tree (7); ceil(nblk / 128) strided partials and the second tree (7,
  clover_trlog_kernel); the host's g0 + g1 (mom_action_total, 1): `sum_depth` = 27 + ceil(nblk / 128) roundings of
  u_d on sum |terms|.  fp32 momenta are squared exactly in double.
* Plaquette (plaquette_site): each leaf is 3 su3_mul_op in T (18, sqrt2 for the complex modulus) on the |U| leaf
  traces; then in double the trace (2) and 3 planes per kind (3); the two trees and the strided partials as above; on
  the host g0 + g1 (1) and / (9 V) (1), and 0.5 (sp + tm) (1) for the total: depth 22 + ceil(nblk / 128).

Where the bounds are loose: the sums add worst-case bounds over every term, while the roundings of V terms cancel like
sqrt(V), so on 16^3 x 32 an fp32 plaquette sits at err/bound ~ 1e-5 (the negative controls show the momentum action's
bound still rejects fp32 site sums by ~10^4); the force's T of a Haar field through 64 paths of 11 links grows like
the product of |U| (spectral radius up to ~1.7) while the force does not, so the table-limit set sits at ~3e-4.  Over
the whole suite the worst err/bound of every family and precision is above 4e-3.
"""
import numpy as np

import clover_build_ref as R
import clover_force_ref as CF
import gauge_cases as G
import precise as PR
import precise_clover as PCL
from quda_b200 import fields as F

U_D = 2.0 ** -53
SQ2 = PR.SQ2
gamma = PCL.gamma
BLOCK = PCL.BLOCK                # kGaugeThreads
K_C1, K_C0, K_ASM = 8, 25, 17
NEWTON_U, SINCOS_U = 4, 4
EXP_SERIES_C1 = 1e-5             # kExpSeriesC1
UPDATE_ORDER = 8                 # kUpdateOrder


def sum_tail(Vh):
    """the summation depth of the two-stage fixed-order reduction over the Vh sites of one parity"""
    nblk = -(-Vh // BLOCK)
    return 7 + -(-nblk // BLOCK) + 7


def mom_action_depth(Vh):
    return 12 + sum_tail(Vh) + 1


def plaquette_depth(Vh):
    return 5 + sum_tail(Vh) + 3


def field_t(prec):
    return np.float64 if prec == 8 else np.float32


def rd(x, prec):
    """x rounded to the kernel's precision, in the reference's real type"""
    return PR.real_t(prec)(field_t(prec)(x))


def mats(mom, prec):
    """mom [..][10] (the values the kernel reads) -> anti-Hermitian [..][3][3] in the reference precision"""
    m = np.asarray(mom).astype(field_t(prec)).astype(PR.real_t(prec))
    out = np.zeros(m.shape[:-1] + (3, 3), PR.cplx_t(prec))
    for n, (i, j) in enumerate(CF.OD):
        out[..., i, j] = m[..., 2 * n] + 1j * m[..., 2 * n + 1]
        out[..., j, i] = -m[..., 2 * n] + 1j * m[..., 2 * n + 1]
    for k in range(3):
        out[..., k, k] = 1j * m[..., 6 + k]
    return out


def traceless(mom, prec, sign=1):
    """(P exactly traceless [..][3][3], the bound of mom_traceless's rounding [..][3][3])"""
    m = np.asarray(mom).astype(field_t(prec)).astype(PR.real_t(prec))
    P = mats(mom, prec)
    tr = (m[..., 6] + m[..., 7] + m[..., 8]) / 3
    u = PR.U_P[prec]
    E = np.zeros(P.shape, np.float64)
    atr = (np.abs(m[..., 6]) + np.abs(m[..., 7]) + np.abs(m[..., 8])).astype(np.float64) / 3
    for k in range(3):
        P[..., k, k] = 1j * (m[..., 6 + k] - tr)
        E[..., k, k] = gamma(3, u) * atr + u * np.abs(m[..., 6 + k] - tr).astype(np.float64)
    return sign * P, E


# ---------------------------------------------------------------------------------------------- force
def ta_bound(m0, f, E, u):
    """per-component bound [..][10] of mom_sub_ta(m0, f) when f [..][3][3] carries the per-part error bound E"""
    af = np.abs(f).astype(np.float64)
    am = np.abs(np.asarray(m0, np.float64))
    b = np.zeros(m0.shape, np.float64)
    for n, (i, j) in enumerate(CF.OD):
        r = 0.5 * (E[..., i, j] + E[..., j, i]) + gamma(2, u) * (0.5 * (af[..., i, j] + af[..., j, i]))
        b[..., 2 * n] = r + gamma(2, u) * am[..., 2 * n]
        b[..., 2 * n + 1] = r + gamma(2, u) * am[..., 2 * n + 1]
    Ed = np.stack([E[..., k, k] for k in range(3)], -1)
    fd = np.stack([np.abs(f[..., k, k].imag).astype(np.float64) for k in range(3)], -1) + Ed
    prop = 2.0 / 3.0 * Ed + (Ed.sum(-1, keepdims=True) - Ed) / 3.0
    rnd = gamma(PCL.K_TA, u) * (am[..., 6:9].max(-1, keepdims=True) + 2 * fd.max(-1, keepdims=True))
    b[..., 6:9] = prop + rnd
    return b


def force(gauge, mom, X, paths, coeffs, eb3, prec):
    """Result of b200_gauge_force: mom [V][4][10] after mom <- TA(mom - eb3 U_mu(x) sum_i c_i path_i); the pad keeps mom's
    value and has bound 0"""
    rt, u = PR.real_t(prec), PR.U_P[prec]
    U = PCL.links(gauge, X, prec)
    aU = np.abs(U).astype(np.float64)
    c = [rd(x, prec) for x in coeffs]
    e = rd(eb3, prec)
    n = len(coeffs)
    f, E = [], []
    for mu in range(4):
        s, Ts = 0, 0
        for i, (ci, p) in enumerate(zip(c, paths[mu])):
            s = s + ci * G.path_field(U, mu, p)
            Ts = Ts + gamma(6 * (len(p) - 1) + (n - i) + 7, u) * abs(float(ci)) * G.path_field(aU, mu, p)
        f.append(R.from_lex(e * (U[mu] @ s), X))
        E.append(R.from_lex(SQ2 * abs(float(e)) * (aU[mu] @ Ts), X))
    f, E = np.stack(f, 1), np.stack(E, 1)          # [V][4][3][3]
    m0 = np.asarray(mom).astype(field_t(prec)).astype(rt)
    ref = PCL.mom_sub_ta(m0, f)
    ref[..., 9] = 0
    bound = ta_bound(m0, f, E, u)
    bound[..., 9] = 0
    return PR.Result(ref, bound)


# ---------------------------------------------------------------------------------------------- the exponential
def invariants(Q):
    """(c0 = Re tr Q^3 / 3, c1 = tr Q^2 / 2) of Hermitian traceless Q [..][3][3]"""
    Q2 = Q @ Q
    return np.einsum("...ij,...ji->...", Q, Q2).real / 3, np.einsum("...ii->...", Q2).real / 2


def exp_coeffs(c0, c1):
    """f_j [3][..] (complex) of exp(iQ) = f0 + f1 Q + f2 Q^2, Morningstar & Peardon's closed form in the arrays'
    precision (c1 > 0), with r = c0 / c0_max clamped to 1 as su3_exp_coeffs does"""
    one = np.ones_like(c1)
    ac0 = np.abs(c0)
    sq = np.sqrt(c1 / 3)
    r = np.minimum(ac0 / (2 * sq ** 3), one)
    theta = np.arccos(r)
    u = sq * np.cos(theta / 3)
    w = np.sqrt(c1) * np.sin(theta / 3)
    w2, u2 = w * w, u * u
    xi0 = np.where(w < 1e-3, 1 - w2 / 6 * (1 - w2 / 20 * (1 - w2 / 42)), np.sin(w) / np.where(w > 0, w, one))
    e2 = np.cos(2 * u) + 1j * np.sin(2 * u)
    em = np.cos(u) - 1j * np.sin(u)
    h0 = (u2 - w2) * e2 + em * (8 * u2 * np.cos(w) + 2j * u * (3 * u2 + w2) * xi0)
    h1 = 2 * u * e2 - em * (2 * u * np.cos(w) - 1j * (3 * u2 - w2) * xi0)
    h2 = e2 - em * (np.cos(w) + 3j * u * xi0)
    den = 9 * u2 - w2
    f = [h0 / den, h1 / den, h2 / den]
    neg = c0 < 0
    return [np.where(neg, (-1) ** j * np.conj(fj), fj) for j, fj in enumerate(f)]


def assemble(f, Q):
    I = np.eye(3, dtype=Q.dtype)
    return f[0][..., None, None] * I + f[1][..., None, None] * Q + f[2][..., None, None] * (Q @ Q)


def expm_taylor(A, order=30):
    """exp(A) [..][3][3] by scaling and squaring a Taylor series, in A's precision"""
    nrm = np.abs(A).astype(np.float64).sum(-1).max(-1)
    s = np.maximum(0, np.ceil(np.log2(np.maximum(nrm, 1e-300) / 0.25))).astype(int)
    smax = int(s.max()) if s.size else 0
    B = A / (2.0 ** s).astype(A.real.dtype)[..., None, None]
    I = np.broadcast_to(np.eye(3, dtype=A.dtype), A.shape)
    E, term = I.copy(), I.copy()
    for k in range(1, order + 1):
        term = term @ B / k
        E = E + term
    for i in range(smax):
        sel = s > i
        E[sel] = E[sel] @ E[sel]
    return E


def expm(A):
    """exp(A) for traceless anti-Hermitian A in A's precision: the closed form where c1 >= 1e-3 (there its own
    cancellation is below 1e-16 u-relative terms), the Taylor series below"""
    Q = -1j * A
    c0, c1 = invariants(Q)
    big = c1 >= 1e-3
    E = expm_taylor(A)
    if big.any():
        E[big] = assemble(exp_coeffs(c0[big], c1[big]), Q[big])
    return E


def _running(x, e):
    return (np.asarray(x, np.float64), np.asarray(e, np.float64))


def sincos_bound(x):
    """sincos_rn with the error of its argument -> ((sin, err), (cos, err))"""
    v, e = x
    err = e + SINCOS_U * U_D
    return (np.sin(v), err), (np.cos(v), err)


def coeff_errors(c0, c1):
    """running bound on the error of su3_exp_coeffs in double at (c0, c1) -> E_f [3][..] (per real part), closed-form
    branch (c1 >= kExpSeriesC1)"""
    u = U_D
    c0, c1 = np.asarray(c0, np.float64), np.asarray(c1, np.float64)
    z = np.zeros_like(c1)
    ac0 = (np.abs(c0), z)
    C1 = (c1, z)
    third = (c1 / 3, u * c1 / 3)
    sqv = np.sqrt(third[0])
    sq = (sqv, third[1] / (2 * np.where(sqv > 0, sqv, 1)) + u * sqv)
    two_sq = (2 * sq[0], 2 * sq[1])
    den_r = PR._mul(two_sq, PR._mul(sq, sq, u), u)
    rv = ac0[0] / den_r[0]
    r = (rv, den_r[1] * rv / den_r[0] + u * rv)
    r = (np.minimum(r[0], 1.0), r[1])
    cv = np.cos(np.arccos(r[0]) / 3)
    c = (cv, r[1] / 6 + NEWTON_U * u)
    uu = PR._mul(sq, c, u)
    one_m = (1 - cv * cv, 2 * cv * c[1] + u * np.abs(1 - cv * cv))
    w2 = PR._mul(C1, one_m, u)
    w2 = (np.maximum(w2[0], 0), w2[1])
    # w enters only through cos w and sin w / w, even functions: their derivatives in w^2 are <= 1/2 and 1/6, so the
    # error of w^2 propagates without the square root's cancellation; the sqrt itself rounds w by u w
    wv = np.sqrt(w2[0])
    u2 = PR._mul(uu, uu, u)
    cw = (np.cos(wv), 0.5 * w2[1] + SINCOS_U * u + u * wv)
    s2u, c2u = sincos_bound((2 * uu[0], 2 * uu[1]))
    su, cu = sincos_bound(uu)
    small = wv < 0.05
    with np.errstate(divide="ignore", invalid="ignore"):
        qv = np.sin(wv) / wv
        q = (qv, w2[1] / 6 + (SINCOS_U * u + u * wv) / wv + u * np.abs(qv))
    ser = (1 - w2[0] / 6, w2[1] / 6 + 4 * u)
    xi0 = (np.where(small, ser[0], np.nan_to_num(q[0])), np.where(small, ser[1], np.nan_to_num(q[1], posinf=0.0)))
    em = (cu, (-su[0], su[1]))
    e2u = (c2u, s2u)
    neg = lambda a: (-a[0], a[1])  # noqa: E731
    sc = lambda a, k: (k * a[0], abs(k) * a[1])  # noqa: E731
    u2mw2 = PR._add(u2, w2, u, sub=True)
    # h0
    t3 = PR._mul(PR._mul(sc(uu, 2.0), PR._add(sc(u2, 3.0), w2, u), u), xi0, u)
    tr, ti = PR._cmul(em, (PR._mul(sc(u2, 8.0), cw, u), t3), u)
    h0 = (PR._add(PR._mul(u2mw2, c2u, 0), tr, u), PR._add(PR._mul(u2mw2, s2u, 0), ti, u))
    # h1
    tr, ti = PR._cmul(em, (PR._mul(sc(uu, 2.0), cw, u), neg(PR._mul(PR._add(sc(u2, 3.0), w2, u, sub=True), xi0, u))), u)
    h1 = (PR._add(PR._mul(sc(uu, 2.0), c2u, 0), tr, u, sub=True),
          PR._add(PR._mul(sc(uu, 2.0), s2u, 0), ti, u, sub=True))
    # h2
    tr, ti = PR._cmul(em, (cw, PR._mul(sc(uu, 3.0), xi0, u)), u)
    h2 = (PR._add(e2u[0], tr, u, sub=True), PR._add(e2u[1], ti, u, sub=True))
    den = PR._add(PR._mul(sc(u2, 9.0), (1.0, 0.0), 0), w2, u, sub=True)
    out = []
    for h in (h0, h1, h2):
        parts = []
        for p in h:
            v = p[0] / den[0]
            parts.append((p[1] + np.abs(v) * den[1]) / den[0] + u * np.abs(v))
        out.append(np.maximum(parts[0], parts[1]))
    return np.stack(out)


def _dF(c0, c1, Q, dc0, dc1):
    """|dF/dc0| dc0 + |dF/dc1| dc1 elementwise [..][3][3] (F = f0 + f1 Q + f2 Q^2), times 2"""
    out = np.zeros(Q.shape, np.float64)
    small = c1 < 1e-3
    out[small] = (dc0[small] + dc1[small])[:, None, None]
    big = ~small
    if big.any():
        a0, a1, Qb = c0[big], c1[big], Q[big]
        h1 = 1e-6 * a1
        d1 = (assemble(exp_coeffs(a0, a1 + h1), Qb) - assemble(exp_coeffs(a0, a1 - h1), Qb)) / (2 * h1)[:, None, None]
        cmax = 2 * np.sqrt(a1 / 3) ** 3
        h0 = 1e-6 * cmax
        base = assemble(exp_coeffs(a0, a1), Qb)
        near = np.abs(a0) + h0 >= cmax
        sgn = np.where(a0 < 0, -1, 1)
        fwd = assemble(exp_coeffs(np.where(near, a0 - sgn * h0, a0 + h0), a1), Qb)
        bwd = assemble(exp_coeffs(np.where(near, a0 - 2 * sgn * h0, a0 - h0), a1), Qb)
        d0 = np.where(near[:, None, None], (3 * base - 4 * fwd + bwd) / (2 * h0)[:, None, None],
                      (fwd - bwd) / (2 * h0)[:, None, None])
        out[big] = 2 * (np.abs(d0).astype(np.float64) * dc0[big][:, None, None]
                        + np.abs(d1).astype(np.float64) * dc1[big][:, None, None])
    return out


class Update:
    """the reference of b200_update_gauge (exact or order 8) and its bound, per link and real component of the
    output links [4][V][3][3][2]"""

    def __init__(self, gauge, mom, X, dt, prec, conj_mom=False, exact=True):
        rt, u = PR.real_t(prec), PR.U_P[prec]
        g = np.asarray(gauge).astype(field_t(prec)).astype(rt)
        U = np.swapaxes(g[..., 0] + 1j * g[..., 1], 0, 1).astype(PR.cplx_t(prec))   # [V][4][3][3]
        aU = np.abs(U).astype(np.float64)
        P, EP = traceless(mom, prec, -1 if conj_mom else 1)
        d = rd(dt, prec)
        if exact:
            ref, bound = self._exact(U, aU, P, EP, d, prec, u)
        else:
            ref, bound = self._order8(U, aU, P, EP, d, dt, prec, u)
        self.result = PR.Result(np.swapaxes(ref, 0, 1), np.swapaxes(bound, 0, 1))

    @staticmethod
    def _exact(U, aU, P, EP, d, prec, u):
        A = d * P
        aA = np.abs(A).astype(np.float64)
        dA = u * aA + abs(float(d)) * EP                               # part 1
        nU = np.linalg.norm(U.astype(np.complex128), 2, axis=(-2, -1))
        part1 = np.sqrt((dA ** 2).sum((-2, -1))) * nU
        Q = -1j * A
        c0, c1 = invariants(Q)
        aQ = np.abs(Q).astype(np.float64)
        aQ2 = aQ @ aQ
        T_c1 = 0.5 * np.einsum("...ii->...", aQ2)
        T_c0 = np.einsum("...ij,...ji->...", aQ, aQ2) / 3
        dc1 = SQ2 * gamma(K_C1, u) * T_c1
        dc0 = SQ2 * gamma(K_C0, u) * T_c0
        dF = _dF(c0, c1, Q, dc0, dc1)                                  # part 2
        f64 = [np.zeros(c1.shape, np.complex128) for _ in range(3)]
        series = np.asarray(c1, np.float64) < EXP_SERIES_C1
        Ef = np.zeros((3,) + c1.shape)
        if (~series).any():
            fb = exp_coeffs(c0[~series], c1[~series])
            for j in range(3):
                f64[j][~series] = fb[j].astype(np.complex128)
            Ef[:, ~series] = coeff_errors(c0[~series], c1[~series])   # part 3
        if series.any():
            a0, a1 = np.asarray(c0[series], np.float64), np.asarray(c1[series], np.float64)
            f64[0][series] = 1 + 1j * a0 * (a1 / 120 - 1 / 6)
            f64[1][series] = a0 / 24 + 1j * (1 - a1 / 6 + a1 ** 2 / 120)
            f64[2][series] = (a1 / 24 - 0.5) + 1j * a0 / 120
            nq = np.linalg.norm(Q[series].astype(np.complex128), 2, axis=(-2, -1))
            trunc = nq ** 6 / 720 * np.exp(nq)
            for j in range(3):
                Ef[j, series] = 3 * U_D * np.abs(f64[j][series]) + (trunc if j == 0 else 0)
        af = [np.abs(x) for x in f64]
        if prec == 4:
            for j in range(3):
                Ef[j] = Ef[j] + u * af[j]
        I = np.eye(3)
        E_coef = (SQ2 * Ef[0])[..., None, None] * I + (SQ2 * Ef[1])[..., None, None] * aQ \
            + (SQ2 * Ef[2])[..., None, None] * aQ2
        T_asm = (af[0][..., None, None] * I + af[1][..., None, None] * aQ + af[2][..., None, None] * aQ2) @ aU
        bound = (part1[..., None, None] + SQ2 * (dF + E_coef) @ aU + SQ2 * gamma(K_ASM, u) * T_asm)
        ref = expm(A) @ U
        return _split(ref), np.repeat(bound[..., None], 2, -1)

    @staticmethod
    def _order8(U, aU, P, EP, d, dt, prec, u):
        rt = PR.real_t(prec)
        aP = np.abs(P).astype(np.float64)
        r, ar, E = U.copy(), aU.copy(), np.zeros(aU.shape)
        for k in range(UPDATE_ORDER, 0, -1):
            sc = d / rt(k)
            sp = sc * P
            asc = abs(float(sc))
            asp = asc * aP
            dsp = 2 * u * asp + asc * EP                               # sc and sc * p rounded, P's trace removal
            r = U + sp @ r
            E = SQ2 * (asp @ E) + SQ2 * (dsp @ ar) + gamma(6, u) * (aU + asp @ ar)
            ar = np.abs(r).astype(np.float64)
        return _split(r), np.repeat(E[..., None], 2, -1)


def _split(m):
    return np.stack([m.real, m.imag], -1)


# ---------------------------------------------------------------------------------------------- the sums
def mom_action(mom, X, prec):
    """Result of b200_mom_action (a scalar)"""
    m = np.asarray(mom).astype(field_t(prec)).astype(np.longdouble)[..., :9]
    terms = (m[..., :6] ** 2).sum(-1) + 0.5 * (m[..., 6:9] ** 2).sum(-1) - 4
    aterm = (m[..., :6] ** 2).sum(-1) + 0.5 * (m[..., 6:9] ** 2).sum(-1) + 4
    ref = terms.sum()
    bound = gamma(mom_action_depth(F.volume_cb(X)), U_D) * float(aterm.sum())
    return PR.Result(np.array([ref]), np.array([bound]))


def plaquette(gauge, X, prec):
    """Result of b200_plaquette: (total, spatial, temporal)"""
    U = PCL.links(gauge, X, prec)
    aU = np.abs(U).astype(np.float64)
    V = int(np.prod(X))
    sums, tsum, asum = {0: 0, 1: 0}, {0: 0.0, 1: 0.0}, {0: 0.0, 1: 0.0}
    for mu, nu in R.PLANES:
        kind = 1 if mu == 3 else 0
        s = lambda a, dm, dn: R.shift(R.shift(a, mu, dm), nu, dn)  # noqa: E731
        P = U[mu] @ s(U[nu], 1, 0) @ R.dag(s(U[mu], 0, 1)) @ R.dag(U[nu])
        Pa = aU[mu] @ s(aU[nu], 1, 0) @ np.swapaxes(s(aU[mu], 0, 1), -1, -2) @ np.swapaxes(aU[nu], -1, -2)
        tr = np.einsum("...ii->...", P).real
        sums[kind] = sums[kind] + tr.sum()
        tsum[kind] += float(np.einsum("...ii->...", Pa).sum())
        asum[kind] += float(np.abs(tr).astype(np.float64).sum())
    u = PR.U_P[prec]
    depth = plaquette_depth(F.volume_cb(X))
    b = [(SQ2 * gamma(18, u) * tsum[k] + gamma(depth, U_D) * (asum[k] + SQ2 * gamma(18, u) * tsum[k])) / (9 * V)
         for k in (0, 1)]
    sp, tm = sums[0] / (9 * V), sums[1] / (9 * V)
    ref = np.array([0.5 * (sp + tm), sp, tm])
    bound = np.array([0.5 * (b[0] + b[1]) + U_D * abs(float(ref[0])), b[0], b[1]])
    return PR.Result(ref, bound)


def assert_scalar(got, res, what):
    """sums: |got - ref| <= bound (the output is double: out_bound adds u_d |ref|)"""
    return PR.assert_within(np.asarray(got, np.float64), res, 8, what)
